// Counter-based RNG for the production (non-parity) sampling mode: Philox4x32-10 keyed by the 64-bit seed, with the
// 64-bit stream id and the 64-bit element counter as its counter words.  Parity tests inject explicit noise tensors
// instead (SURVEY.md §7 "RNG parity"), so this generator never has to match torch's.
//
// Stream plan.  Every draw site takes its stream id from one of the stream_* functions below and nowhere else.  Ids
// below 2^32 are the ones earlier releases drew from, kept so that a seed keeps producing the same output; each kind
// leaves them for its own tagged range, (tag << 32) | sub, exactly where its legacy ids would run into another kind's.
// The legacy ranges are disjoint:
//   mel x_T (q_sample, or ProDiff's randn)     1000                                  counter ti*80 + c
//   mel reverse step t < 999                   1001 + t                 (else tag 2) counter ti*80 + c
//   F0 x_T, net n                              2000 + 100000 n                       counter ti
//   F0 Gaussian step t < 4000, net n           2010 + 100000 n + 2 t    (else tag 4 + n) counter ti
//   F0 uniform (Gumbel) step t < 4000, net n   2011 + 100000 n + 2 t    (else tag 6 + n) counter 2*ti + j
//   vocoder NSF initial phase, utterance b < 8224  0x5151 + b          (else tag 8) counter h (harmonic 1..8)
//   vocoder NSF source noise                   0x7171                                counter ti*9 + h
// i.e. [1000, 2000), [2000, 10010), [20817, 29041), 29041, [102000, 110010), and every tagged id is >= 2^32, so no two
// kinds share a stream whatever T, the batch size or the utterance index.  ti is the counter row: row0 + the row (frame,
// or sample for the vocoder source) inside the utterance, and b the initial-phase stream index, both from the
// utterance's entry of the layout's key table (UttRng, common.cuh), whose key is the Philox key of its draws.
//
// Batch composition.  With injected noise every utterance's result is independent of the batch it is in.  The key
// table has two fillings (upload_layout), and the streams above are the same in both:
//   one seed per call (Seq::seed): key = seed, row0 = the utterance's tight offset in the call, stream index b = the
//     utterance's index, so an utterance draws different noise in a different batch.  The persistent mel groups
//     (ssb_model_set_persistent_groups) key group g by seed + 0x9E3779B97F4A7C15 g and count rows inside the group;
//   one seed per utterance (Seq::utt_seeds, the ssb_*_keyed entries): key = utt_seeds[b], row0 = 0, stream index 0,
//     i.e. exactly the draws of a B = 1 call with seed utt_seeds[b] (which is group 0 of itself), whatever the batch.
#pragma once
#include <stdint.h>

namespace ssb {

__host__ __device__ constexpr uint64_t philox_stream(uint64_t tag, uint32_t sub) { return (tag << 32) | sub; }
__host__ __device__ constexpr uint64_t stream_mel_xt() { return 1000; }
__host__ __device__ constexpr uint64_t stream_mel_step(int t) { return t < 999 ? 1001 + (uint64_t)t : philox_stream(2, (uint32_t)t); }
__host__ __device__ constexpr uint64_t stream_f0_xt(int net) { return 2000 + 100000 * (uint64_t)net; }
__host__ __device__ constexpr uint64_t stream_f0_gauss(int net, int t) {
  return t < 4000 ? stream_f0_xt(net) + 10 + 2 * (uint64_t)t : philox_stream(4 + net, (uint32_t)t);
}
__host__ __device__ constexpr uint64_t stream_f0_unif(int net, int t) {
  return t < 4000 ? stream_f0_xt(net) + 11 + 2 * (uint64_t)t : philox_stream(6 + net, (uint32_t)t);
}
__host__ __device__ constexpr uint64_t stream_voc_ini(int b) { return b < 8224 ? 0x5151 + (uint64_t)b : philox_stream(8, (uint32_t)b); }
__host__ __device__ constexpr uint64_t stream_voc_src() { return 0x7171; }

__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
  const uint32_t hi0 = __umulhi(M0, c[0]), lo0 = M0 * c[0];
  const uint32_t hi1 = __umulhi(M1, c[2]), lo1 = M1 * c[2];
  const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
__device__ __forceinline__ void philox4(uint64_t seed, uint64_t stream, uint64_t ctr, uint32_t (&out)[4]) {
  uint32_t c[4] = {(uint32_t)ctr, (uint32_t)(ctr >> 32), (uint32_t)stream, (uint32_t)(stream >> 32)};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3];
}
// (k + 0.5) / 2^24 for k = x >> 8, in fp32: (0, 1].  For k = 2^24 - 1 the sum 16777215.5 rounds up to 2^24, i.e. 1.
__device__ __forceinline__ float u32_to_unit_closed(uint32_t x) { return ((x >> 8) + 0.5f) * (1.0f / 16777216.0f); }
// Uniform draws, (0, 1): the one value that rounds up to 1 is clamped to 1 - 2^-24, every other one is the value
// earlier releases drew.
__device__ __forceinline__ float u32_to_unit(uint32_t x) { return fminf(u32_to_unit_closed(x), 0.99999994039535522461f); }
__device__ __forceinline__ float philox_uniform(uint64_t seed, uint64_t stream, uint64_t idx) {
  uint32_t o[4];
  philox4(seed, stream, idx, o);
  return u32_to_unit(o[0]);
}
// Box-Muller on the (0, 1] grid: u1 = 1 gives radius 0, a finite draw (the radius at the top of the grid), so the
// normals keep exactly the values earlier releases drew.
__device__ __forceinline__ float philox_normal(uint64_t seed, uint64_t stream, uint64_t idx) {
  uint32_t o[4];
  philox4(seed, stream, idx, o);
  const float u1 = u32_to_unit_closed(o[0]), u2 = u32_to_unit_closed(o[1]);
  return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}

}  // namespace ssb
