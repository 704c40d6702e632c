// wgmma / TMA implicit-GEMM conv1d for the dense contractions of the denoisers (SURVEY.md §8 a13/a18).
//
// Precision: every fp32 operand is carried as TWO fp16 planes (hi = fp16(x), lo = fp16(x - hi));
// each K step issues three wgmma (hi*hi + hi*lo + lo*hi) into one fp32 register accumulator (SURVEY.md §7: single-pass
// bf16/fp16/TF32 cannot meet the mel L-inf < 1e-3 bar at T=100; a 3-pass split can).  Effective tensor peak = 1/3 of the
// fp16 peak.  The split is exact to about 2^-22 of x only while lo is a normal fp16 number, |x| >= 2^-3, and exists only
// for |x| < 65520 (hi = inf above).  So:
//  * weights: the packer splits w * 2^s with one power of two per tensor, s = 14 - ceil(log2 max|w|) (ConvTC::wscale =
//    2^-s, applied in the epilogue as fmaf(acc, wscale, bias)): about 22 bits at any weight magnitude, for every weight
//    above max|w| * 2^-16;
//  * activations: relative 2^-22 for |a| >= 2^-3, below that an absolute error floor of 2^-25 per element (lo is
//    subnormal), and defined only for |a| < 65520;
//  * single_pass: 2^-12 relative (one fp16 rounding) on the weights at any magnitude, the same activation range.
//
// Layout: A = activation planes [rows, C] fp16 row-major (guard-banded rows, see common.cuh), loaded by
// TMA as [128 rows x 64 ch] boxes with 128B swizzle at row offset (tap - center) * dilation;
// B = weights [taps*N, Cin] fp16 (K-major), boxes [64 n x 64 ch] (single-CTA kernel) or [hb x 64] (CTA-pair kernel:
// each CTA of a 2-CTA cluster loads its own 128 rows of A and half of a 2*hb-wide weight tile, multicast to both CTAs;
// hb = 64 when N % 128 == 0, else 32).  CTAs are persistent over the tiles.  The pair kernel is used when there are
// >= num_SMs pair tiles (ceil(ntiles / 2) * N / (2 hb)), the single-CTA kernel with 64-wide N tiles otherwise
// (conv_gemm_tc()).
// single_pass (GemmTC): one wgmma per K step on the hi planes alone, i.e. the operands rounded once to fp16 (~11 mantissa
// bits) with fp32 accumulation; the lo planes are not read.  A speed / accuracy choice of the mel denoiser and the vocoder
// (ssb_model_set_mel_precision, ssb_vocoder_set_precision), not the default.
// 3-tap convs at pair sizes take the tap-reuse variant: one halo-extended activation tile per K block serves all three taps.
// Pair launches from different streams are ordered against each other on the device (conv_gemm_tc.cu).
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "conv_gemm.cuh"

namespace ssb {

struct ConvTC {            // packed weights for the tensor-core path
  __half* W_hi = nullptr;  // [taps][N][Cin]
  __half* W_lo = nullptr;
  CUtensorMap tm_hi[2], tm_lo[2];  // weight boxes of [0]: 64 rows, [1]: 32 rows
  int hb = 0;                       // CTA-pair kernel: weight rows each CTA of a pair loads (half of a 2*hb-wide N tile)
  int taps = 1, Cin = 0, N = 0, dil = 1, center = 0;
  const float* bias = nullptr;  // [N] (packed column order)
  float wscale = 1.0f;          // the planes hold W * 2^s; wscale = 2^-s multiplies the accumulator (pack_conv_tc)
  bool ok = false;
};

// The skip accumulator (RES_SKIP) and the conditioner addend (GATE) are touched once per launch: they are read and written
// with ld/st.global.cs (evict-first), so that they do not push the y / z planes (re-read by the next launch) out of L2.
struct EpiTC {
  int mode = EPI_GENERIC;        // EPI_GENERIC: out = acc + bias ; EPI_GATE ; EPI_RES_SKIP
  const float* bias = nullptr;
  float* out = nullptr;          // GENERIC / RES_SKIP residual path: fp32 [rows, ldo]
  int ldo = 0;
  __half* oh = nullptr;          // GATE: z planes [rows, C];  RES_SKIP: y = x_new + vec2 planes [rows, C] (may be null)
  __half* ol = nullptr;
  int ldh = 0;
  const float* add = nullptr;    // GATE: pre-activation addend [rows, ld_add] in packed (sigmoid, tanh) column order - the
  int ld_add = 0;                //   hoisted, step-invariant conditioner projection of this layer (stages.cu prepare_cond)
  const float* res = nullptr;    // RES_SKIP: x [rows, ld_res]
  int ld_res = 0;
  const __half* rh = nullptr;    // RES_SKIP, planes-only residual stream: x = (rh + rl) - vec1 is read from the fp16 hi/lo
  const __half* rl = nullptr;    //   planes of y = x + step bias (the GATE GEMM's own A operand); no fp32 x is read or written
  int ld_rh = 0;
  const float* vec1 = nullptr;   //   step bias of the CURRENT layer [C]
  float beta = 1.0f;
  const float* vec2 = nullptr;   // RES_SKIP: step bias of the next layer [C]
  float* skip = nullptr;         // RES_SKIP: [rows, ld_skip]
  int ld_skip = 0;
  int C = 0;
  int skip_init = 0;
  // EPI_GENERIC extras: v = act(acc + bias); v += res; out = accum ? (out + v) * gamma : v; planes = plane_act(v)
  int act = ACT_NONE;
  float act_slope = 0.1f;
  int accum = 0;
  float gamma = 1.0f;
  int plane_act = ACT_NONE;      // activation applied to the value written to the fp16 planes (pre-activation of the consumer)
  float plane_slope = 0.1f;
  float alpha = 1.0f;            // GENERIC: v = act((acc + bias) * alpha)   (ACT_GELU supported here for the FFT FFN)
  const float* rowmask = nullptr;  // GENERIC: v = (v + res) * rowmask[row]
  int n_valid = 0;               // > 0: output columns >= n_valid are padding (weights padded to a tile multiple): skipped
  int skip_tiled = 0;            // RES_SKIP: skip accumulator stored chunk-tiled - [row tile][32-row quarter][32-col chunk][32 rows][32 cols]
                                 //   fp32, so that every 32 x 32 epilogue chunk is one contiguous 4 KB block (private to this epilogue)
  int out_nb = 0;                // GENERIC, > 0: `out` is column-block-major: block j = columns [j*out_nb, (j+1)*out_nb) is its own
  int64_t out_bs = 0;            //   [rows, out_nb] matrix at out + j * out_bs (the hoisted conditioner: one matrix per layer)
  __half* sh = nullptr;          // RES_SKIP (last layer): the finished skip sum also as fp16 planes [rows, C]
  __half* sl = nullptr;
};

struct GemmTC {
  const __half* A_hi = nullptr;  // [rows_total, Cin]
  const __half* A_lo = nullptr;
  int64_t rows_total = 0;
  const ConvTC* w = nullptr;
  const int2* tiles = nullptr;
  int ntiles = 0;
  EpiTC e;
  bool single_pass = false;  // true: hi*hi only (A_lo and W_lo unread); false: the 3-pass hi/lo split
};

bool tc_available();  // driver entry point for cuTensorMapEncodeTiled resolved
int make_weight_maps(ConvTC* w);
// TMA descriptor of an activation plane [rows, cols] fp16 (box 128 rows x 64 cols, 128B swizzle)
int make_act_map(CUtensorMap* m, const void* ptr, int64_t rows, int cols, int box_rows = 128);
int conv_gemm_tc(Ctx& ctx, const GemmTC& p);
// diagnostics: launches of one kernel variant ("tc2<64,GATE>", "tc<64,GENERIC>", ...), the variants seen so far,
// and the activation-descriptor cache counters
long long variant_launch_count(const char* name);
int variant_names(char* buf, int cap);
void tensor_map_cache_stats(long long* encodes, long long* hits);
// x fp32 [rows, ld] -> hi/lo planes [rows, C] (all rows incl. guards; guards stay zero)
int split_planes(Ctx& ctx, const float* x, int ld, int64_t rows, int C, float scale, __half* hi, __half* lo);

}  // namespace ssb
