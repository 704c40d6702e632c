// Vocoder output denoiser: denoise(wav, v) of the reference (tasks/tts/vocoder_infer/hifigan_nsf.py:14-22), which
// HifiGAN.spec2wav (:73-74) runs on the generator's waveform when hparams['vocoder_denoise_c'] > 0:
//     S  = librosa.stft(wav, n_fft, hop, win, window="hann", center=True, pad_mode="constant")
//     S' = max(|S| - v, 0) * exp(i angle(S))                    (= S * max(0, 1 - v / |S|), 0 where |S| = 0)
//     y  = librosa.istft(S', hop, win, window="hann", center=True)
// As kernels, on the guard-banded ragged layout with one row per STFT frame (an utterance of n = F hop samples has F + 1):
//   1. the forward DFT is the implicit-GEMM STFT of the mel front-end (frontend.cu): the waveform as rows of hop samples, the
//      zero guard rows are the constant centre padding, one taps = span / hop conv with N = 2 nbp columns (re | im);
//   2. k_spec_subtract scales every bin by max(0, 1 - v / |S|) (straight into the fp16 hi/lo A planes of the next GEMM on
//      the tensor-core path);
//   3. irfft, window and overlap-add are ONE implicit-GEMM conv over the frame rows: output row r holds trimmed samples
//      [r hop, (r + 1) hop), which frames r - taps/2 + 1 .. r + taps/2 overlap, so it is a taps-tap conv with Cin = 2 nbp,
//      N = hop and the synthesis basis of each tap's window segment as weights (guard rows = absent frames);
//   4. k_istft_unpack divides by the window sum-square of the frames 0 .. F that exist and writes the tight output.
// Bins are padded to a multiple of 32 so that 2 nbp meets the tensor-core kernel's Cin % 64 / N % 64 (1024 -> 544).
#include <float.h>

#include <cmath>

#include <memory>
#include <vector>

#include "../../include/stylesinger_b200.h"
#include "conv_gemm.cuh"
#include "model.cuh"
#include "stages.cuh"

struct ssb_wav_denoise {
  ssb::DevicePool pool;
  ssb::Conv fwd;       // [taps][hop][2 nbp]: analysis basis (re | im), window folded in
  ssb::Conv inv;       // [taps][2 nbp][hop]: synthesis basis (irfft x window) of each tap's frame segment
  ssb::ConvTC fwd_tc, inv_tc;  // the same weights for the tensor-core kernel (ok == false when not eligible)
  float* wsq = nullptr;        // [span] squared window at frame sample i - lead (0 outside the window)
  int n_fft = 0, hop = 0, win = 0, nbins = 0, nbp = 0, taps = 0;
  int tc_mode = 0;  // 0: fp32 FFMA GEMMs; 1: tensor cores for batches of >= 8 row tiles (the default); 2: tensor cores always
};

namespace ssb {

namespace {

// S * max(0, 1 - v / |S|) for the bins < nbins of every frame row; the output's padding bins and guard rows stay zero
__global__ void k_spec_subtract(const int4* utt, const float* spec, int ld, int nbp, int nbins, float v, float* out,
                                __half* oh, __half* ol) {
  const int b = blockIdx.y;
  const int4 u = utt[b];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)u.y * nbins) return;
  const int64_t t = i / nbins;
  const int k = (int)(i - t * nbins);
  const int64_t o = ((int64_t)u.x + t) * ld + k;
  const float re = spec[o], im = spec[o + nbp];
  const float mag = hypotf(re, im);
  const float g = mag > 0.f ? fmaxf(0.f, 1.f - v / mag) : 0.f;  // np.angle(0) = 0: a zero bin stays zero
  const float a = re * g, c = im * g;
  if (oh) {
    const __half ah = __float2half_rn(a), ch = __float2half_rn(c);
    oh[o] = ah; ol[o] = __float2half_rn(a - __half2float(ah));
    oh[o + nbp] = ch; ol[o + nbp] = __float2half_rn(c - __half2float(ch));
  } else {
    out[o] = a; out[o + nbp] = c;
  }
}

// overlap-added rows [rows, hop] -> tight output: trimmed sample i = r hop + c of an utterance with F + 1 frames divided by
// sum_t w^2[i + n_fft/2 - t hop] over its frames t = 0 .. F where that sum exceeds tiny(float32) (librosa.istft)
__global__ void k_istft_unpack(const int4* utt, const int32_t* sample_offs, const float* y, const float* wsq, int hop, int taps,
                               float* out) {
  const int b = blockIdx.y;
  const int4 u = utt[b];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)(u.y - 1) * hop) return;  // the row behind the last sample is not part of the output
  const int r = (int)(i / hop);
  const int c = (int)(i - (int64_t)r * hop);
  const int cen = taps / 2 - 1;  // tap k reads frame r + k - cen at frame row taps - 1 - k
  float ss = 0.f;
  for (int k = 0; k < taps; ++k) {
    const int t = r + k - cen;
    if (t >= 0 && t < u.y) ss += wsq[(taps - 1 - k) * hop + c];
  }
  float a = y[((int64_t)u.x + r) * hop + c];
  if (ss > FLT_MIN) a /= ss;
  out[(int64_t)sample_offs[b] + i] = a;
}

int check_lengths(const int32_t* sample_offsets, int B, int hop) {
  SSB_CHECK(sample_offsets && B >= 0, "bad argument");
  for (int b = 0; b < B; ++b) {
    const int64_t n = (int64_t)sample_offsets[b + 1] - sample_offsets[b];
    SSB_CHECK(n > 0 && n % hop == 0, "every utterance length must be a positive multiple of hop_size");
  }
  return 0;
}

// [taps][Cin][N] fp32 -> tensor-core packing (torch layout [N][Cin][taps] for pack_conv_tc)
int pack_tc(DevicePool& pool, const std::vector<float>& W, int taps, int Cin, int N, int center, ConvTC* out) {
  std::vector<float> t((size_t)N * Cin * taps);
  for (int j = 0; j < taps; ++j)
    for (int c = 0; c < Cin; ++c)
      for (int n = 0; n < N; ++n) t[((size_t)n * Cin + c) * taps + j] = W[((size_t)j * Cin + c) * N + n];
  HostTensor ht;
  ht.data = t.data();
  ht.shape = {N, Cin, taps};
  RUN(pack_conv_tc(pool, &ht, 1, PACK_PLAIN, nullptr, out));
  out->center = center;
  return 0;
}

int run_denoise(Ctx& c, const ssb_wav_denoise& d, const Seq& q, const float* wav, const int32_t* sample_offsets_host, int B,
                float v, float* out) {
  SeqDev s;
  RUN(upload_layout(c, q, 1, &s));
  const int N2 = 2 * d.nbp;
  const bool tc = d.tc_mode == 2 || (d.tc_mode == 1 && s.ntiles >= 8);  // long_batch_tc's threshold (stages.cu)
  int32_t* offs_dev = c.alloc<int32_t>((size_t)B + 1);
  float* rows = alloc_rows(c, s, d.hop);  // zero-filled incl. guards = the constant centre padding
  float* spec = alloc_rows(c, s, N2, false);
  float* y = alloc_rows(c, s, d.hop, false);
  float* sub = nullptr;
  __half *wh = nullptr, *wl = nullptr, *sh = nullptr, *sl = nullptr;
  if (tc) {
    wh = c.alloc<__half>((size_t)s.rows * d.hop);
    wl = c.alloc<__half>((size_t)s.rows * d.hop);
    sh = c.alloc<__half>((size_t)s.rows * N2);
    sl = c.alloc<__half>((size_t)s.rows * N2);
  } else {
    sub = alloc_rows(c, s, N2);  // zero-filled: the inverse GEMM reads the guard rows as absent frames
  }
  WS_OK(c);
  if (c.dry || B == 0) return 0;
  if (tc) {  // zero-filled for the same reason
    SSB_CUDA(cudaMemsetAsync(sh, 0, (size_t)s.rows * N2 * sizeof(__half), c.stream));
    SSB_CUDA(cudaMemsetAsync(sl, 0, (size_t)s.rows * N2 * sizeof(__half), c.stream));
  }
  SSB_CUDA(cudaMemcpyAsync(offs_dev, sample_offsets_host, sizeof(int32_t) * ((size_t)B + 1), cudaMemcpyHostToDevice, c.stream));
  RUN(wav_rows(c, s, offs_dev, wav, d.hop, rows));
  if (tc) {
    RUN(split_planes(c, rows, d.hop, s.rows, d.hop, 1.0f, wh, wl));
    GemmTC g = make_gemm_tc(d.fwd_tc, s, wh, wl);
    g.e.out = spec; g.e.ldo = N2;
    RUN(conv_gemm_tc(c, g));
  } else {
    ConvGemm g = make_gemm(d.fwd, s, rows, d.hop);
    g.e.out = spec; g.e.ldo = N2;
    RUN(conv_gemm(c, g));
  }
  {
    const int64_t per = (int64_t)s.maxlen * d.nbins;
    k_spec_subtract<<<dim3((unsigned)((per + 255) / 256), (unsigned)B), 256, 0, c.stream>>>(s.utt, spec, N2, d.nbp, d.nbins, v, sub,
                                                                                           sh, sl);
    SSB_CUDA(cudaGetLastError());
    ++g_launches;
  }
  // irfft's 1 / n_fft is the epilogue's alpha, not folded into the synthesis weights: n_fft need not be a power of two,
  // and a rounded product in the weights would change the FFMA path's bits (the tensor-core packing scales its planes by
  // a power of two of its own, so it would not need it)
  const float inv_n = 1.0f / (float)d.n_fft;
  if (tc) {
    GemmTC g = make_gemm_tc(d.inv_tc, s, sh, sl);
    g.e.alpha = inv_n; g.e.out = y; g.e.ldo = d.hop;
    RUN(conv_gemm_tc(c, g));
  } else {
    ConvGemm g = make_gemm(d.inv, s, sub, N2);
    g.e.alpha = inv_n; g.e.out = y; g.e.ldo = d.hop;
    RUN(conv_gemm(c, g));
  }
  {
    const int64_t per = (int64_t)(s.maxlen - 1) * d.hop;
    k_istft_unpack<<<dim3((unsigned)((per + 255) / 256), (unsigned)B), 256, 0, c.stream>>>(s.utt, offs_dev, y, d.wsq, d.hop, d.taps,
                                                                                          out);
    SSB_CUDA(cudaGetLastError());
    ++g_launches;
  }
  return 0;
}

}  // namespace

}  // namespace ssb

using namespace ssb;

extern "C" {

int ssb_wav_denoise_create(ssb_wav_denoise_t** out, int32_t fft_size, int32_t hop_size, int32_t win_length) {
  SSB_CHECK(out, "null argument");
  *out = nullptr;
  SSB_CHECK(fft_size > 0 && hop_size > 0 && win_length > 0 && win_length <= fft_size, "bad denoiser geometry");
  SSB_CHECK(fft_size % 2 == 0 && hop_size % 16 == 0, "the implicit-GEMM STFT needs an even n_fft and hop_size a multiple of 16");
  const int span = stft_span(fft_size, hop_size);
  SSB_CHECK(span / hop_size / 2 <= GUARD, "n_fft / hop_size too large for the guard band");
  std::unique_ptr<ssb_wav_denoise> d(new ssb_wav_denoise);
  d->n_fft = fft_size; d->hop = hop_size; d->win = win_length;
  d->nbins = fft_size / 2 + 1;
  d->nbp = (d->nbins + 31) & ~31;
  d->taps = span / hop_size;
  const int N2 = 2 * d->nbp, T = d->taps;
  const std::vector<float> Wf = dft_basis(fft_size, hop_size, win_length, d->nbp, false);  // [span][N2] = [taps][hop][N2]
  const std::vector<float> Bi = dft_basis(fft_size, hop_size, win_length, d->nbp, true);
  // inverse tap k reads frame r + k - (taps/2 - 1), whose row r is frame row taps - 1 - k: W[k][col][c] = Bi[(taps-1-k) hop + c][col]
  std::vector<float> Wi((size_t)span * N2);
  for (int k = 0; k < T; ++k)
    for (int col = 0; col < N2; ++col)
      for (int c = 0; c < hop_size; ++c)
        Wi[((size_t)k * N2 + col) * hop_size + c] = Bi[((size_t)(T - 1 - k) * hop_size + c) * N2 + col];
  const std::vector<double> w = hann_window(fft_size, win_length);
  const int lead = (span - fft_size) / 2;
  std::vector<float> wsq((size_t)span, 0.f);
  for (int j = 0; j < fft_size; ++j) wsq[(size_t)(j + lead)] = (float)(w[(size_t)j] * w[(size_t)j]);
  d->fwd.W = d->pool.upload(Wf);
  d->fwd.taps = T; d->fwd.Cin = hop_size; d->fwd.N = N2; d->fwd.Npad = N2; d->fwd.dil = 1; d->fwd.center = T / 2;
  d->inv.W = d->pool.upload(Wi);
  d->inv.taps = T; d->inv.Cin = N2; d->inv.N = hop_size; d->inv.Npad = hop_size; d->inv.dil = 1; d->inv.center = T / 2 - 1;
  d->wsq = d->pool.upload(wsq);
  SSB_CHECK(d->fwd.W && d->inv.W && d->wsq, "device allocation failed");
  RUN(pack_tc(d->pool, Wf, T, hop_size, N2, d->fwd.center, &d->fwd_tc));
  RUN(pack_tc(d->pool, Wi, T, N2, hop_size, d->inv.center, &d->inv_tc));
  d->tc_mode = d->fwd_tc.ok && d->inv_tc.ok ? 1 : 0;
  *out = d.release();
  return 0;
}

void ssb_wav_denoise_free(ssb_wav_denoise_t* d) { delete d; }

size_t ssb_wav_denoise_workspace_bytes(const ssb_wav_denoise_t* d, const int32_t* sample_offsets, int32_t B) {
  if (!d || check_lengths(sample_offsets, B, d->hop) != 0) return 0;
  Ctx c;
  c.dry = true;
  Seq q;
  if (build_seq(sample_offsets, B, d->hop, &q) != 0) return 0;
  if (run_denoise(c, *d, q, nullptr, sample_offsets, B, 0.f, nullptr) != 0) return 0;
  return c.high;
}

int ssb_wav_denoise_forward(const ssb_wav_denoise_t* d, const float* wav_in, const int32_t* sample_offsets, int32_t B, float v,
                            float* wav_out, void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(d && wav_in && sample_offsets && wav_out && workspace && B >= 0, "bad argument");
  SSB_CHECK(std::isfinite(v) && v >= 0.f, "the denoising strength v must be finite and >= 0");
  RUN(check_lengths(sample_offsets, B, d->hop));
  Ctx c;
  c.base = (char*)workspace; c.cap = workspace_bytes; c.stream = (cudaStream_t)stream;
  Seq q;
  RUN(build_seq(sample_offsets, B, d->hop, &q));
  return run_denoise(c, *d, q, wav_in, sample_offsets, B, v, wav_out);
}

int ssb_wav_denoise_set_tensor_cores(ssb_wav_denoise_t* d, int32_t enable) {
  SSB_CHECK(d, "null denoiser");
  SSB_CHECK(enable >= 0 && enable <= 2, "enable must be 0, 1 or 2");
  d->tc_mode = d->fwd_tc.ok && d->inv_tc.ok ? enable : 0;
  return d->tc_mode;
}

}  // extern "C"
