// Common definitions for the stylesinger_b200 CUDA library (sm_90a only).
//
// Data layout used by every kernel in this library ("guard-banded ragged rows"):
//   * activations are channels-last fp32 matrices [rows, C];
//   * a batch of B utterances with lengths L_b is stored as ONE row-major matrix in which utterance b
//     occupies rows [rs_b, rs_b + L_b), rs_0 = G, rs_{b+1} = rs_b + L_b + G  (G = guard rows);
//   * rows that belong to no utterance (guards, tail slack) are ZERO and are never written, so a
//     conv tap that reaches past either end of an utterance reads the zero "same" padding the
//     reference's Conv1d(padding=...) would supply, with no per-element bounds logic and no
//     cross-utterance leakage (true-length semantics, SURVEY.md §7 "Batched semantics");
//   * a time-upsampled view (vocoder stages) uses the same table with every row index multiplied by
//     the rate m (rs_b*m, L_b*m, G*m), so [rows, u*C] of stage i IS [rows*u, C] of stage i+1.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <string>
#include <vector>

namespace ssb {

constexpr int GUARD = 16;        // guard rows at rate 1 (>= max conv reach at rate 1: DiffNet dilation 8)
constexpr int TAIL_SLACK = 256;  // rows appended so that a partially valid tile can over-read safely
constexpr int TILE_M = 128;      // rows per GEMM tile

extern std::atomic<long long> g_launches;  // kernels launched by this library (diagnostic; see ssb_launch_count)
void set_error(const std::string& msg);
const char* last_error();

#define SSB_CHECK(cond, msg)                                                     \
  do {                                                                           \
    if (!(cond)) {                                                               \
      ssb::set_error(std::string(msg) + " (" #cond ") at " __FILE__ ":" +        \
                     std::to_string(__LINE__));                                  \
      return -1;                                                                 \
    }                                                                            \
  } while (0)

#define SSB_CUDA(call)                                                           \
  do {                                                                           \
    cudaError_t e_ = (call);                                                     \
    if (e_ != cudaSuccess) {                                                     \
      ssb::set_error(std::string("CUDA error: ") + cudaGetErrorString(e_) +      \
                     " in " #call " at " __FILE__ ":" + std::to_string(__LINE__)); \
      return -2;                                                                 \
    }                                                                            \
  } while (0)

// ---------------------------------------------------------------------------------------------
// Ragged layout (host side description + device tile table)
// ---------------------------------------------------------------------------------------------
struct Seq {
  int B = 0;
  std::vector<int> len;   // L_b at rate 1
  std::vector<int> rs;    // row start at rate 1
  int64_t rows1 = 0;      // (rs_{B-1} + L_{B-1} + G): rows at rate 1 excluding slack
  int64_t total = 0;      // sum L_b
  int maxlen = 0;
  // Philox keys of the layout's draws (philox.cuh, "Batch composition"): utt_seeds (host [B]) keys utterance b by
  // utt_seeds[b] and counts its rows from 0; NULL keys every utterance by `seed` and counts the tight rows of the layout.
  uint64_t seed = 0;
  const uint64_t* utt_seeds = nullptr;

  void build(const int32_t* offsets, int B_) {
    B = B_;
    len.resize(B);
    rs.resize(B);
    int64_t r = GUARD;
    total = 0;
    maxlen = 0;
    for (int b = 0; b < B; ++b) {
      len[b] = offsets[b + 1] - offsets[b];
      rs[b] = (int)r;
      r += len[b] + GUARD;
      total += len[b];
      if (len[b] > maxlen) maxlen = len[b];
    }
    rows1 = r;
  }
  int64_t rows(int rate = 1) const { return rows1 * rate + TAIL_SLACK; }
  int ntiles(int rate = 1) const {
    int n = 0;
    for (int b = 0; b < B; ++b) n += (len[b] * rate + TILE_M - 1) / TILE_M;
    return n;
  }
};

// Philox key and counter base of one utterance: its row t (at the layout's rate) draws with counter row row0 + t, and
// its vocoder initial phase from stream_voc_ini(ini) (philox.cuh).
struct UttRng {
  uint64_t key;
  int32_t row0;
  int32_t ini;
};

// Device-side view of one layout at one rate.
struct SeqDev {
  const int2* tiles = nullptr;  // (row0, nvalid) per 128-row tile
  int ntiles = 0;
  const int4* utt = nullptr;    // per utterance: (row_start, len, tight_offset, 0) at this rate
  const UttRng* rng = nullptr;  // per utterance: Philox key and counter base at this rate
  int B = 0;
  int64_t rows = 0;             // allocated rows (incl. slack)
  int64_t total = 0;            // tight rows
  int maxlen = 0;
  int rate = 1;
  const int4* tile_pos = nullptr;  // per tile: (tight index of its first row, utterance, first row inside it, 0)
};

// ---------------------------------------------------------------------------------------------
// Workspace bump allocator. In "dry" mode nothing is launched and only the high-water mark is
// computed, so ssb_*_workspace_bytes() runs the very same planning code as the real call.
// ---------------------------------------------------------------------------------------------
struct Ctx {
  char* base = nullptr;
  size_t cap = 0;
  size_t off = 0;
  size_t high = 0;
  bool dry = false;
  bool failed = false;
  cudaStream_t stream = 0;

  void* alloc_bytes(size_t n) {
    size_t a = (off + 255) & ~size_t(255);
    off = a + n;
    if (off > high) high = off;
    if (dry) return (void*)(uintptr_t)256;  // non-null dummy
    if (off > cap) {
      failed = true;
      return nullptr;
    }
    return base + a;
  }
  template <typename T>
  T* alloc(size_t count) { return (T*)alloc_bytes(count * sizeof(T)); }
  size_t mark() const { return off; }
  void release(size_t m) { off = m; }
};

// zero-filled fp32 matrix in a layout
float* alloc_rows(Ctx& c, const SeqDev& s, int C, bool zero = true);
int upload_layout(Ctx& c, const Seq& s, int rate, SeqDev* out);

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float softplusf_(float x) { return x > 20.0f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float mishf_(float x) { return x * tanhf(softplusf_(x)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace ssb
