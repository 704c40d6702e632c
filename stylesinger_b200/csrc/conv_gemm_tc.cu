// wgmma + TMA implicit-GEMM conv1d for Hopper (see conv_gemm_tc.cuh).  sm_90a only.
//
// CTA = 384 threads, persistent over (M-tile, N-tile) pairs:
//   warp 0 (1 lane)  TMA producer: per K block loads A_hi, A_lo [128x64] and W_hi, W_lo [BNx64] (128B swizzle)
//   warps 4-11       two consumer warpgroups: each issues the 3-product wgmma chain (M64 N=BN K16, fp32 accumulators in
//                    registers) for its 64 rows, then runs the fused epilogue through shared-memory transpose buffers
// PASSES = 1 (single-pass fp16, GemmTC::single_pass): the producer loads only the A_hi / W_hi tiles and each K step issues
// one wgmma (hi*hi); the stage layout and the epilogue are those of PASSES = 3, so the lo halves of each stage stay unused.
// smem ring: BN=128: 3 stages x 64 KB, BN=64: 4 stages x 48 KB; mbarriers full/empty per stage.  The single-CTA kernel
// (BN=64) serves problems too small to fill the GPU with pairs.  The CTA-pair variant (cluster of 2, BN = 2 hb = 64 or 128)
// gives each CTA its own row tile and one half of a shared weight tile, which TMA multicasts into both CTAs.
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <unordered_map>

#include "conv_gemm_tc.cuh"
#include "tc_common.cuh"

namespace ssb {

namespace {

constexpr int BM = 128, BK = 64;
constexpr int A_TILE = BM * BK * 2;  // 16 KB
constexpr int EPI_WARPS = 8;                       // two consumer warpgroups
constexpr int NTHREADS = 128 + 32 * EPI_WARPS;
constexpr int XPOSE_BYTES = EPI_WARPS * 32 * 32 * 4;  // epilogue transpose buffers: one [32 x 32] fp32 per warp

constexpr int HALO = 8;                     // largest dilation served by the tap-reuse variant (DiffNet: 1, 2, 4, 8)
constexpr int A3_ROWS = BM + 2 * HALO;      // 144
constexpr int A3_TILE = A3_ROWS * BK * 2;   // 18 KB per plane (a multiple of 1024: swizzle pattern alignment)
constexpr int ASLOTS = 2;                   // tap-reuse activation ring

template <int BN, bool REUSE>
struct Cfg {
  static constexpr int B_TILE = BN * BK * 2;
  static constexpr int STAGE = REUSE ? 2 * B_TILE : 2 * A_TILE + 2 * B_TILE;  // REUSE: weights only
  static constexpr int STAGES = BN == 128 ? 3 : 4;
  static constexpr int ARING = REUSE ? ASLOTS * 2 * A3_TILE : 0;
  static constexpr int SMEM = ARING + STAGES * STAGE + XPOSE_BYTES + 1024 + 256;
  static_assert(SMEM <= 227 * 1024, "exceeds the 227 KB of shared memory a Hopper block can have");
};

struct TCParams {
  const int2* tiles;
  int ntiles, NT, taps, kchunks, dil, center, N;
  float wscale;  // ConvTC::wscale: the accumulator holds the contraction with W * 2^s; the epilogue multiplies it by 2^-s
  EpiTC e;
};

using namespace tc;

// ---- epilogue ------------------------------------------------------------------------------------------------
// The wgmma accumulator fragment scatters a row over four lanes in pairs of columns.  Storing from that mapping makes
// every warp store touch many 128-byte lines with 8-byte pieces.  So each pair of consumer warps writes its 32 rows, 64
// columns at a time, into two 4 KB shared-memory buffers (float4 chunks XOR-swizzled by row) and each warp then works on
// one [32 x 32] chunk in a COALESCED mapping:
// step i of 8 handles rows 4i + lane/8, columns 4*(lane%8) .. +3, i.e. every warp access covers 4 full 128-byte lines.

struct Pre {
  float4 a[8];  // epilogue global operands (residual / skip) of the 8 steps of one chunk, fetched ahead of use
};

// rows of this warp: r0 + [0, 32); nrows valid ones.  Lane's row in step i: 4i + (lane >> 3); columns n4 .. n4+3.
// Loads are UNCONDITIONAL (rows past the end of an utterance lie inside the guard band / tail slack of every buffer, and
// their values are never stored) and walk one pointer with a constant step: the first version spent more instructions on
// per-access 64-bit address arithmetic and row predicates than on the epilogue itself (profiles/r02_epilogue_sass_v9.md).
template <int MODE>
__device__ __forceinline__ void prefetch_chunk(const EpiTC& e, int64_t r0, int nrows, int n, int lane, Pre& p, int tq) {
  (void)nrows;
  if (e.n_valid > 0 && n >= e.n_valid) return;
  const int rq = lane >> 3, q4 = (lane & 7) * 4;
  const float* src = nullptr;
  int64_t st = 0;  // floats between consecutive steps (4 rows)
  bool once = false;  // data this launch reads exactly once and nobody re-reads soon: streaming (evict-first) loads
  if constexpr (MODE == EPI_GENERIC) {
    if (!e.res) return;
    src = e.res + (r0 + rq) * e.ld_res + n + q4; st = 4 * (int64_t)e.ld_res;
  } else if constexpr (MODE == EPI_RES_SKIP) {
    if (n < e.C) {
      if (e.rh) {  // residual stream carried as fp16 hi/lo planes: 4 columns = 8 bytes per plane, packed into one float4
        const __half* ph = e.rh + (r0 + rq) * e.ld_rh + n + q4;
        const __half* pl = e.rl + (r0 + rq) * e.ld_rh + n + q4;
        const int64_t sth = 4 * (int64_t)e.ld_rh;
#pragma unroll
        for (int i = 0; i < 8; ++i, ph += sth, pl += sth) {
          const uint2 h = *reinterpret_cast<const uint2*>(ph);
          const uint2 l = *reinterpret_cast<const uint2*>(pl);
          p.a[i] = make_float4(__uint_as_float(h.x), __uint_as_float(h.y), __uint_as_float(l.x), __uint_as_float(l.y));
        }
        return;
      }
      src = e.res + (r0 + rq) * e.ld_res + n + q4; st = 4 * (int64_t)e.ld_res;
    } else if (!e.skip_init) {
      if (e.skip_tiled) {  // chunk (tq, (n - C) / 32) is a contiguous [32 rows][32 cols] block
        src = e.skip + ((int64_t)tq * (e.C >> 5) + ((n - e.C) >> 5)) * 1024 + rq * 32 + q4; st = 128;
      } else {
        src = e.skip + (r0 + rq) * e.ld_skip + (n - e.C) + q4; st = 4 * (int64_t)e.ld_skip;
      }
      once = true;
    } else return;
  } else {  // EPI_GATE: the hoisted conditioner projection of this layer
    if (!e.add) return;
    src = e.add + (r0 + rq) * e.ld_add + n + q4; st = 4 * (int64_t)e.ld_add;
    once = true;
  }
  if (once) {
#pragma unroll
    for (int i = 0; i < 8; ++i, src += st) p.a[i] = __ldcs(reinterpret_cast<const float4*>(src));
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i, src += st) p.a[i] = *reinterpret_cast<const float4*>(src);  // one 64-bit add per step
  }
}

// hi/lo split of 4 (2) values as packed words - computed OUTSIDE the row predicate so that a chunk's 8 steps stay one basic
// block (only the store instructions are predicated) and the scheduler can interleave the steps' dependent chains
__device__ __forceinline__ void split_pack4(float a, float b, float c, float d, uint2& uh, uint2& ul) {
  const __half2 h0 = __floats2half2_rn(a, b), h1 = __floats2half2_rn(c, d);
  const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
  const __half2 l0 = __floats2half2_rn(a - f0.x, b - f0.y), l1 = __floats2half2_rn(c - f1.x, d - f1.y);
  uh.x = *reinterpret_cast<const uint32_t*>(&h0); uh.y = *reinterpret_cast<const uint32_t*>(&h1);
  ul.x = *reinterpret_cast<const uint32_t*>(&l0); ul.y = *reinterpret_cast<const uint32_t*>(&l1);
}
__device__ __forceinline__ void split_pack2(float a, float b, uint32_t& uh, uint32_t& ul) {
  const __half2 h0 = __floats2half2_rn(a, b);
  const float2 f0 = __half22float2(h0);
  const __half2 l0 = __floats2half2_rn(a - f0.x, b - f0.y);
  uh = *reinterpret_cast<const uint32_t*>(&h0);
  ul = *reinterpret_cast<const uint32_t*>(&l0);
}
// One 32 x 32 accumulator chunk (columns [n, n+32)) of this warp, already in its transpose buffer: the fused epilogue.
// MODE is a template parameter (and the chunk loop is not unrolled) to keep the epilogue's code small: the first
// version carried all three modes x 4-8 unrolled chunks = 13k SASS instructions and ran out of the instruction cache.
// Everything that does not depend on the step (pointers, flags, slopes) is hoisted into registers: the epilogue warps
// run alone on their scheduler, so every instruction and every constant-bank reload is exposed latency.
__device__ __forceinline__ float act_slope_of(int act, float slope) {  // act(v) == fmaxf(v, v * s) for s in [0, 1]
  return act == ACT_RELU ? 0.0f : (act == ACT_LRELU ? slope : 1.0f);
}
template <int MODE>
__device__ __forceinline__ void epilogue_chunk(const EpiTC& e, float ws, const float4* xb, int64_t r0, int nrows, int n,
                                               int lane, const Pre& pre, int tq) {
  if (e.n_valid > 0 && n >= e.n_valid) return;  // warp-uniform
  const int q = lane & 7, rq = lane >> 3;  // step i: row rq + 4i, columns n4 .. n4 + 3
  const int n4 = n + 4 * q;
  const int64_t rb = r0 + rq;
  const float4* xr = xb + rq * 8;          // row rq + 4i, chunk q ^ ((rq + 4i) & 7) = (q ^ rq) ^ (4 * (i & 1))
  const int qx = q ^ rq;
  float b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
  if (e.bias) {
    const float4 bv = __ldg(reinterpret_cast<const float4*>(e.bias + n4));
    b0 = bv.x; b1 = bv.y; b2 = bv.z; b3 = bv.w;
  }
  // acc * ws + bias is one fmaf: ws is a power of two, so it costs no instruction over acc + bias and rounds once.
  // Everything below is computed for all 8 steps; only the STORES are predicated on the row being valid (i < nsteps).
  const int nsteps = nrows > rq ? (nrows - rq + 3) >> 2 : 0;
  if constexpr (MODE == EPI_GATE) {
    const int64_t st = 4 * (int64_t)e.ldh;
    __half* ph = e.oh + rb * e.ldh + (n4 >> 1);
    __half* pl = e.ol + rb * e.ldh + (n4 >> 1);
    const bool has_add = e.add != nullptr;
#pragma unroll
    for (int i = 0; i < 8; ++i, ph += st, pl += st) {
      const float4 acc = xr[i * 32 + (qx ^ (4 * (i & 1)))];
      float g0 = fmaf(acc.x, ws, b0), f0 = fmaf(acc.y, ws, b1), g1 = fmaf(acc.z, ws, b2), f1 = fmaf(acc.w, ws, b3);
      if (has_add) {
        const float4 ad = pre.a[i];
        g0 += ad.x; f0 += ad.y; g1 += ad.z; f1 += ad.w;
      }
      uint32_t zh, zl;
      split_pack2(gate_act(g0, f0), gate_act(g1, f1), zh, zl);
      if (i < nsteps) {
        *reinterpret_cast<uint32_t*>(ph) = zh;
        *reinterpret_cast<uint32_t*>(pl) = zl;
      }
    }
  } else if constexpr (MODE == EPI_RES_SKIP) {
    if (n < e.C) {
      const float beta = e.beta;
      float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
      const bool planes = e.oh != nullptr;
      if (planes && e.vec2) {
        const float4 sv = __ldg(reinterpret_cast<const float4*>(e.vec2 + n4));
        s0 = sv.x; s1 = sv.y; s2 = sv.z; s3 = sv.w;
      }
      const bool res_planes = e.rh != nullptr, has_out = e.out != nullptr;
      float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;  // step bias of the current layer: x = (hi + lo) - c
      if (res_planes && e.vec1) {
        const float4 cv = __ldg(reinterpret_cast<const float4*>(e.vec1 + n4));
        c0 = cv.x; c1 = cv.y; c2 = cv.z; c3 = cv.w;
      }
      float* po = has_out ? e.out + rb * e.ldo + n4 : nullptr;
      const int64_t sto = 4 * (int64_t)e.ldo, sth = 4 * (int64_t)e.ldh;
      __half* ph = planes ? e.oh + rb * e.ldh + n4 : nullptr;
      __half* pl = planes ? e.ol + rb * e.ldh + n4 : nullptr;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 acc = xr[i * 32 + (qx ^ (4 * (i & 1)))];
        float4 x0 = pre.a[i];
        if (res_planes) {  // (hi0 hi1 | hi2 hi3 | lo0 lo1 | lo2 lo3) as raw half2 bits
          const uint32_t u0 = __float_as_uint(x0.x), u1 = __float_as_uint(x0.y), u2 = __float_as_uint(x0.z), u3 = __float_as_uint(x0.w);
          const float2 h01 = __half22float2(*reinterpret_cast<const __half2*>(&u0)), h23 = __half22float2(*reinterpret_cast<const __half2*>(&u1));
          const float2 l01 = __half22float2(*reinterpret_cast<const __half2*>(&u2)), l23 = __half22float2(*reinterpret_cast<const __half2*>(&u3));
          x0 = make_float4((h01.x + l01.x) - c0, (h01.y + l01.y) - c1, (h23.x + l23.x) - c2, (h23.y + l23.y) - c3);
        }
        const float v0 = (fmaf(acc.x, ws, b0) + x0.x) * beta, v1 = (fmaf(acc.y, ws, b1) + x0.y) * beta;
        const float v2 = (fmaf(acc.z, ws, b2) + x0.z) * beta, v3 = (fmaf(acc.w, ws, b3) + x0.w) * beta;
        uint2 yh, yl;
        split_pack4(v0 + s0, v1 + s1, v2 + s2, v3 + s3, yh, yl);
        const bool ok = i < nsteps;
        if (ok && has_out) *reinterpret_cast<float4*>(po) = make_float4(v0, v1, v2, v3);
        if (ok && planes) {
          *reinterpret_cast<uint2*>(ph) = yh;
          *reinterpret_cast<uint2*>(pl) = yl;
        }
        po += sto; ph += sth; pl += sth;
      }
    } else {
      const int sc = n4 - e.C;
      const bool init = e.skip_init != 0;
      const bool planes = e.sh != nullptr;
      float* ps = e.skip_tiled ? e.skip + ((int64_t)tq * (e.C >> 5) + ((n - e.C) >> 5)) * 1024 + rq * 32 + 4 * q
                               : e.skip + rb * e.ld_skip + sc;
      const int64_t sts = e.skip_tiled ? 128 : 4 * (int64_t)e.ld_skip, sth = 4 * (int64_t)e.C;
      __half* ph = planes ? e.sh + rb * e.C + sc : nullptr;
      __half* pl = planes ? e.sl + rb * e.C + sc : nullptr;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 acc = xr[i * 32 + (qx ^ (4 * (i & 1)))];
        float v0 = fmaf(acc.x, ws, b0), v1 = fmaf(acc.y, ws, b1), v2 = fmaf(acc.z, ws, b2), v3 = fmaf(acc.w, ws, b3);
        if (!init) {
          const float4 o = pre.a[i];
          v0 += o.x; v1 += o.y; v2 += o.z; v3 += o.w;
        }
        const bool ok = i < nsteps;
        if (ok) __stcs(reinterpret_cast<float4*>(ps), make_float4(v0, v1, v2, v3));
        if (planes) {  // last layer only
          uint2 kh, kl;
          split_pack4(v0, v1, v2, v3, kh, kl);
          if (ok) {
            *reinterpret_cast<uint2*>(ph) = kh;
            *reinterpret_cast<uint2*>(pl) = kl;
          }
        }
        ps += sts; ph += sth; pl += sth;
      }
    }
  } else {  // EPI_GENERIC: v = act(acc + bias) (+ res); out = accum ? (out + v) * gamma : v; planes = plane_act(v + vec2)
    const float sa = act_slope_of(e.act, e.act_slope), sp = act_slope_of(e.plane_act, e.plane_slope);
    const bool gelu = e.act == ACT_GELU;
    const float alpha = e.alpha;
    const float* rmask = e.rowmask ? e.rowmask + rb : nullptr;
    const bool has_res = e.res != nullptr, has_out = e.out != nullptr, accum = e.accum != 0, planes = e.oh != nullptr;
    const float gamma = e.gamma;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    if (planes && e.vec2) {
      const float4 sv = __ldg(reinterpret_cast<const float4*>(e.vec2 + n4));
      s0 = sv.x; s1 = sv.y; s2 = sv.z; s3 = sv.w;
    }
    float* po = has_out ? e.out + rb * e.ldo + n4 : nullptr;
    int64_t sto = 4 * (int64_t)e.ldo;
    const int64_t sth = 4 * (int64_t)e.ldh;
    if (has_out && e.out_nb > 0) {  // column-block-major output (one [rows, out_nb] matrix per block of columns)
      const int blk = n4 / e.out_nb;
      po = e.out + (int64_t)blk * e.out_bs + rb * e.out_nb + (n4 - blk * e.out_nb);
      sto = 4 * (int64_t)e.out_nb;
    }
    __half* ph = planes ? e.oh + rb * e.ldh + n4 : nullptr;
    __half* pl = planes ? e.ol + rb * e.ldh + n4 : nullptr;
    // MRF accumulation reads `out` back: all 8 rows up front (one exposed round trip per chunk instead of one per step - the
    // compiler cannot move a load above the previous step's store to the same array)
    float4 oacc[8];
    if (has_out && accum) {
      const float* pr = po;
#pragma unroll
      for (int i = 0; i < 8; ++i, pr += sto) oacc[i] = *reinterpret_cast<const float4*>(pr);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 acc = xr[i * 32 + (qx ^ (4 * (i & 1)))];
      float v0 = fmaf(acc.x, ws, b0) * alpha, v1 = fmaf(acc.y, ws, b1) * alpha, v2 = fmaf(acc.z, ws, b2) * alpha,
            v3 = fmaf(acc.w, ws, b3) * alpha;
      if (gelu) {
        v0 = gelu_erf(v0); v1 = gelu_erf(v1); v2 = gelu_erf(v2); v3 = gelu_erf(v3);
      } else {
        v0 = fmaxf(v0, v0 * sa); v1 = fmaxf(v1, v1 * sa); v2 = fmaxf(v2, v2 * sa); v3 = fmaxf(v3, v3 * sa);
      }
      if (has_res) {
        const float4 x0 = pre.a[i];
        v0 += x0.x; v1 += x0.y; v2 += x0.z; v3 += x0.w;
      }
      if (rmask) {
        const float mk = rmask[4 * i];
        v0 *= mk; v1 *= mk; v2 *= mk; v3 *= mk;
      }
      if (has_out && accum) {
        const float4 o = oacc[i];
        v0 = (v0 + o.x) * gamma; v1 = (v1 + o.y) * gamma; v2 = (v2 + o.z) * gamma; v3 = (v3 + o.w) * gamma;
      }
      const bool ok = i < nsteps;
      if (ok && has_out) *reinterpret_cast<float4*>(po) = make_float4(v0, v1, v2, v3);
      if (planes) {
        const float w0 = v0 + s0, w1 = v1 + s1, w2 = v2 + s2, w3 = v3 + s3;
        uint2 qh, ql;
        split_pack4(fmaxf(w0, w0 * sp), fmaxf(w1, w1 * sp), fmaxf(w2, w2 * sp), fmaxf(w3, w3 * sp), qh, ql);
        if (ok) {
          *reinterpret_cast<uint2*>(ph) = qh;
          *reinterpret_cast<uint2*>(pl) = ql;
        }
      }
      po += sto; ph += sth; pl += sth;
    }
  }
}

// TMA loads of an operand's hi plane and, with NPL == 2, of its lo plane `stride` bytes further
template <int NPL>
__device__ __forceinline__ void tma_load_planes(uint32_t dst, uint32_t stride, const CUtensorMap* hi, const CUtensorMap* lo,
                                                uint32_t bar, int c0, int c1) {
  tma_load_2d(dst, hi, bar, c0, c1);
  if constexpr (NPL == 2) tma_load_2d(dst + stride, lo, bar, c0, c1);
}

// REUSE (3-tap convs, centre tap 1, dilation <= HALO): per K block ONE halo-extended activation tile of
// BM + 2 HALO rows is loaded into its own ring, and the three taps read it through wgmma descriptors whose start address
// is moved by whole 128-byte rows (the 128B swizzle phase follows the shared-memory address, and the tile starts on a
// 1024-byte boundary).  Per tap only the weight tile is loaded: a third of the activation bytes of the plain variant.
template <int BN, int CL, int MODE, bool REUSE, int PASSES>
__global__ void __launch_bounds__(NTHREADS, 1)
conv_gemm_wg_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                    const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
                    const TCParams p) {
  using K = Cfg<BN, REUSE>;
  constexpr int STAGES = K::STAGES;
  constexpr int HB = BN / CL;  // weight rows this CTA loads per K block (CL == 2: and multicasts to its peer)
  constexpr int NCH = BN / 32;
  static_assert(PASSES == 3 || PASSES == 1, "3-pass hi/lo split or single-pass fp16");
  constexpr int NPL = PASSES == 3 ? 2 : 1;  // fp16 planes loaded per operand
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // [activation ring (REUSE)][stage ring][transpose buffers][barriers]
  float* xpose = reinterpret_cast<float*>(smem + K::ARING + STAGES * K::STAGE);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + K::ARING + STAGES * K::STAGE + XPOSE_BYTES);
  const uint32_t abase = smem_u32(smem), sbase = abase + K::ARING;
  const uint32_t full0 = smem_u32(bars), empty0 = full0 + 8 * STAGES, afull0 = empty0 + 8 * STAGES, aempty0 = afull0 + 8 * ASLOTS;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = CL > 1 ? cluster_rank() : 0u;
  const int cid = (int)blockIdx.x / CL, ncl = (int)gridDim.x / CL;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, CL * EPI_WARPS);  // every consumer warp of every CTA that receives this stage's weights
    }
    for (int s = 0; s < ASLOTS; ++s) {
      mbar_init(afull0 + 8 * s, 1);
      mbar_init(aempty0 + 8 * s, EPI_WARPS);      // activation tiles are this CTA's own
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (CL > 1) cluster_sync_all();  // both CTAs' barriers initialised before any multicast or remote arrive
  else __syncthreads();

  const int total = (CL > 1 ? (p.ntiles + 1) / 2 : p.ntiles) * p.NT;
  const int nk = p.taps * p.kchunks;

  if (warp < 4) {  // warpgroup 0 only runs the TMA producer: its registers go to the consumer warpgroups
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == 0 && lane == 0) {
      int stage = 0, as = 0;
      uint32_t phase = 0, aph = 0;
      // weight tile (or this CTA's half of it, multicast to the pair) of one K block into stage `stage`
      auto load_b = [&](const CUtensorMap* mb_h, const CUtensorMap* mb_l, int c0, int brow, uint32_t extra_bytes) {
        mbar_wait(empty0 + 8 * stage, phase ^ 1);
        const uint32_t fb = full0 + 8 * stage;
        mbar_expect_tx(fb, NPL * K::B_TILE + extra_bytes);
        const uint32_t sb = sbase + stage * K::STAGE + (REUSE ? 0u : (uint32_t)(2 * A_TILE));
        if (CL > 1) {
          const uint32_t boff = rank * (uint32_t)(HB * BK * 2);
          tma_load_2d_mc(sb + boff, mb_h, fb, c0, brow + (int)rank * HB, (uint16_t)3);
          if constexpr (PASSES == 3) tma_load_2d_mc(sb + K::B_TILE + boff, mb_l, fb, c0, brow + (int)rank * HB, (uint16_t)3);
        } else {
          tma_load_2d(sb, mb_h, fb, c0, brow);
          if constexpr (PASSES == 3) tma_load_2d(sb + K::B_TILE, mb_l, fb, c0, brow);
        }
        return fb;
      };
      for (int tile = cid; tile < total; tile += ncl) {
        const int mq = tile / p.NT, nt = tile - mq * p.NT;
        int mt = CL * mq + (int)rank;
        if (mt >= p.ntiles) mt = CL * mq;  // odd tile count: the peer re-loads the leader's rows and writes nothing
        const int row0 = p.tiles[mt].x;
        if constexpr (REUSE) {
          for (int kc = 0; kc < p.kchunks; ++kc) {
            mbar_wait(aempty0 + 8 * as, aph ^ 1);
            const uint32_t ab = afull0 + 8 * as, sa = abase + as * (2 * A3_TILE);
            mbar_expect_tx(ab, NPL * A3_TILE);
            tma_load_planes<NPL>(sa, A3_TILE, &tmA_hi, &tmA_lo, ab, kc * BK, row0 - HALO);
            if (++as == ASLOTS) { as = 0; aph ^= 1; }
            for (int tap = 0; tap < 3; ++tap) {
              load_b(&tmB_hi, &tmB_lo, kc * BK, tap * p.N + nt * BN, 0u);
              if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
          }
        } else {
          for (int kb = 0; kb < nk; ++kb) {
            const int tap = kb / p.kchunks;
            const int c0 = (kb - tap * p.kchunks) * BK;
            const int arow = row0 + (tap - p.center) * p.dil;
            // the expect_tx of load_b also covers this CTA's activation boxes of the same stage
            const uint32_t fb = load_b(&tmB_hi, &tmB_lo, c0, tap * p.N + nt * BN, (uint32_t)(NPL * A_TILE));
            const uint32_t sa = sbase + stage * K::STAGE;
            tma_load_planes<NPL>(sa, A_TILE, &tmA_hi, &tmA_lo, fb, c0, arow);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    __syncwarp();
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    // Two consumer warpgroups; warpgroup cw owns accumulator rows [64 cw, 64 cw + 64).  For the epilogue the warps pair up:
    // pair ew (warps 4 + 2 ew, 5 + 2 ew) holds rows [32 ew, 32 ew + 32) and stages them, 64 columns at a time, into two
    // [32 x 32] transpose buffers; warp parity eg then runs the fused epilogue on chunk 2 cp + eg of that pair of chunks.
    const int cw = (warp - 4) >> 2;
    const int ew = (warp - 4) >> 1;
    const int eg = warp & 1;
    float* xb_pair = xpose + ew * 2048;
    const uint32_t pair_bar = 1u + (uint32_t)ew;
    const uint32_t peer_empty0 = CL > 1 ? mapa_u32(empty0, rank ^ 1u) : 0u;
    int stage = 0, as = 0;
    uint32_t phase = 0, aph = 0;
    float acc[BN / 2];
    auto release_b = [&](int st) {  // this warp has finished reading stage st (in both CTAs' counts when CL == 2)
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(empty0 + 8 * st);
        if (CL > 1) mbar_arrive_cluster(peer_empty0 + 8 * st);
      }
    };
    auto mma_block = [&](uint64_t dah, uint64_t dal, uint64_t dbh, uint64_t dbl) {
      wg_fence();
      fence_acc(acc);
#pragma unroll
      for (int ks = 0; ks < BK / 16; ++ks) {
        const uint64_t off = (uint64_t)((ks * 32) >> 4);  // 16 fp16 = 32 bytes along K inside the swizzle atom
        if constexpr (BN == 128) {
          wgmma_n128(acc, dah + off, dbh + off, 1u);
          if constexpr (PASSES == 3) {
            wgmma_n128(acc, dah + off, dbl + off, 1u);
            wgmma_n128(acc, dal + off, dbh + off, 1u);
          }
        } else {
          wgmma_n64(acc, dah + off, dbh + off, 1u);
          if constexpr (PASSES == 3) {
            wgmma_n64(acc, dah + off, dbl + off, 1u);
            wgmma_n64(acc, dal + off, dbh + off, 1u);
          }
        }
      }
      wg_commit();
      fence_acc(acc);
      wg_wait<1>();  // the MMAs of the previous K block are done: its stage can be refilled
      fence_acc(acc);
    };
    for (int tile = cid; tile < total; tile += ncl) {
      const int mq = tile / p.NT, nt = tile - mq * p.NT;
      const int mt = CL * mq + (int)rank;
      const int2 t = mt < p.ntiles ? p.tiles[mt] : make_int2(0, 0);
      const int64_t r0 = (int64_t)t.x + ew * 32;
      const int nrows = min(32, max(0, t.y - ew * 32));
      const int tq = mt * 4 + ew;
      const int n0 = nt * BN;
      Pre cur, nxt;
      if (nrows > 0) prefetch_chunk<MODE>(p.e, r0, nrows, n0 + eg * 32, lane, cur, tq);  // overlaps the MMAs
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      if constexpr (REUSE) {
        for (int kc = 0; kc < p.kchunks; ++kc) {
          mbar_wait(afull0 + 8 * as, aph);
          const uint32_t sa = abase + as * (2 * A3_TILE) + cw * 8192;
          for (int tap = 0; tap < 3; ++tap) {
            mbar_wait(full0 + 8 * stage, phase);
            const uint32_t sb = sbase + stage * K::STAGE;
            const uint32_t sh = (uint32_t)(HALO + (tap - 1) * p.dil) * 128u;  // whole rows
            mma_block(make_sdesc(sa + sh), make_sdesc(sa + A3_TILE + sh), make_sdesc(sb), make_sdesc(sb + K::B_TILE));
            if (prev >= 0) release_b(prev);
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
          wg_wait<0>();  // all three taps have read the activation tile
          fence_acc(acc);
          release_b(prev);
          prev = -1;
          __syncwarp();
          if (lane == 0) mbar_arrive(aempty0 + 8 * as);
          if (++as == ASLOTS) { as = 0; aph ^= 1; }
        }
      } else {
        for (int kb = 0; kb < nk; ++kb) {
          mbar_wait(full0 + 8 * stage, phase);
          const uint32_t sa = sbase + stage * K::STAGE;
          mma_block(make_sdesc(sa + cw * 8192), make_sdesc(sa + A_TILE + cw * 8192), make_sdesc(sa + 2 * A_TILE),
                    make_sdesc(sa + 2 * A_TILE + K::B_TILE));
          if (prev >= 0) release_b(prev);
          prev = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wg_wait<0>();
        fence_acc(acc);
        if (prev >= 0) release_b(prev);
      }
      const int rbase = 16 * (warp & 1) + (lane >> 2);
#pragma unroll
      for (int cp = 0; cp < BN / 64; ++cp) {
#pragma unroll
        for (int nb = 0; nb < 8; ++nb) {
          float* xb = xb_pair + (nb >> 2) * 1024;
          const int cc = 8 * (nb & 3) + 2 * (lane & 3);  // column inside the 32-wide chunk
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int rr = rbase + 8 * h;
            const int j = 4 * (8 * cp + nb) + 2 * h;
            *reinterpret_cast<float2*>(xb + (rr * 8 + ((cc >> 2) ^ (rr & 7))) * 4 + (cc & 3)) = make_float2(acc[j], acc[j + 1]);
          }
        }
        named_sync(pair_bar, 64);
        const int ch = 2 * cp + eg;
        if (ch + 2 < NCH && nrows > 0) prefetch_chunk<MODE>(p.e, r0, nrows, n0 + (ch + 2) * 32, lane, nxt, tq);
        if (nrows > 0)
          epilogue_chunk<MODE>(p.e, p.wscale, reinterpret_cast<float4*>(xb_pair + eg * 1024), r0, nrows, n0 + ch * 32, lane, cur,
                              tq);
        cur = nxt;
        named_sync(pair_bar, 64);  // both chunks consumed before the buffers are refilled
      }
    }
  }
  if (CL > 1) cluster_sync_all();  // neither CTA may exit while its peer still multicasts into it or arrives on its barriers
}

__global__ void k_split_planes(const float* x, int ld, int64_t rows, int C, float scale, __half* hi, __half* lo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * C) return;
  const int64_t r = i / C;
  const int c = (int)(i - r * C);
  const float v = x[r * ld + c] * scale;
  const __half h = __float2half_rn(v);
  hi[i] = h;
  lo[i] = __float2half_rn(v - __half2float(h));
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
std::mutex g_host_mu;  // guards the driver entry point, the per-device kernel attributes and the descriptor cache

EncodeTiledFn get_encode() {
  static std::atomic<EncodeTiledFn> fn_cached{nullptr};
  static std::atomic<bool> tried{false};
  if (!tried.load(std::memory_order_acquire)) {
    std::lock_guard<std::mutex> lk(g_host_mu);
    if (!tried.load(std::memory_order_relaxed)) {
      void* fn = nullptr;
      cudaDriverEntryPointQueryResult q;
      if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess &&
          q == cudaDriverEntryPointSuccess)
        fn_cached.store((EncodeTiledFn)fn, std::memory_order_relaxed);
      tried.store(true, std::memory_order_release);
    }
  }
  return fn_cached.load(std::memory_order_relaxed);
}

// 2-D fp16 row-major [rows, cols] tensor, box [box_rows x 64 cols], 128B swizzle, zero OOB fill
int make_map(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  EncodeTiledFn enc = get_encode();
  SSB_CHECK(enc != nullptr, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * sizeof(__half)};
  cuuint32_t box[2] = {(cuuint32_t)BK, box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult rc = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SSB_CHECK(rc == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed");
  return 0;
}

// Activation descriptors are a pure function of (pointer, rows, cols, box): a sampler loop re-launches the same GEMMs
// on the same workspace buffers T x L times, so they are encoded once and looked up afterwards (VERDICT r1 weak #7).
struct MapKey {
  const void* ptr; uint64_t rows; uint32_t cols, box;
  bool operator==(const MapKey& o) const { return ptr == o.ptr && rows == o.rows && cols == o.cols && box == o.box; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    uint64_t h = (uint64_t)(uintptr_t)k.ptr * 0x9E3779B97F4A7C15ull;
    h ^= (k.rows + 0x7F4A7C15u) * 0xC2B2AE3D27D4EB4Full;
    h ^= ((uint64_t)k.cols << 32 | k.box) * 0x165667B19E3779F9ull;
    return (size_t)(h ^ (h >> 29));
  }
};
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_map_cache;
long long g_map_encodes = 0, g_map_hits = 0;

int cached_act_map(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  const MapKey k{ptr, rows, (uint32_t)cols, box_rows};
  std::lock_guard<std::mutex> lk(g_host_mu);
  auto it = g_map_cache.find(k);
  if (it != g_map_cache.end()) {
    *m = it->second;
    ++g_map_hits;
    return 0;
  }
  if (g_map_cache.size() > 8192) g_map_cache.clear();  // bounded: workspaces move when a batch shape changes
  if (make_map(m, ptr, rows, cols, box_rows)) return -1;
  g_map_cache.emplace(k, *m);
  ++g_map_encodes;
  return 0;
}

// Kernel attributes (cudaFuncSetAttribute) and the SM count are PER DEVICE: one process may drive several GPUs.
constexpr int MAX_DEV = 64;
int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev >= 0 && dev < MAX_DEV ? dev : 0;
}
int device_sms() {
  static std::atomic<int> sms[MAX_DEV];
  const int dev = current_device();
  int n = sms[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
    sms[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}
template <typename KernelT>
int configure_once(KernelT kernel, std::atomic<bool>* done /*[MAX_DEV]*/, int smem) {
  const int dev = current_device();
  if (done[dev].load(std::memory_order_acquire)) return 0;
  std::lock_guard<std::mutex> lk(g_host_mu);
  if (!done[dev].load(std::memory_order_relaxed)) {
    SSB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    done[dev].store(true, std::memory_order_release);
  }
  return 0;
}

// Per-variant launch counters (ssb_variant_launch_count): lets a test assert WHICH kernel a problem size took.
struct VariantCounter { const char* name; std::atomic<long long> n; };
VariantCounter g_variants[48];
std::atomic<int> g_nvariants{0};
std::atomic<long long>* variant_counter(const char* name) {
  std::lock_guard<std::mutex> lk(g_host_mu);
  const int n = g_nvariants.load();
  for (int i = 0; i < n; ++i)
    if (strcmp(g_variants[i].name, name) == 0) return &g_variants[i].n;
  if (n >= 48) return &g_variants[47].n;
  g_variants[n].name = name;
  g_variants[n].n.store(0);
  g_nvariants.store(n + 1);
  return &g_variants[n].n;
}
const char* mode_name(int mode) { return mode == EPI_GATE ? "GATE" : (mode == EPI_RES_SKIP ? "RES_SKIP" : "GENERIC"); }

// index into ConvTC::tm_hi / tm_lo of the weight descriptor whose box has `rows` rows
constexpr int map_index(int rows) { return rows == 64 ? 0 : 1; }
// Cluster (CTA-pair) kernels from DIFFERENT streams are ordered against each other on the device: two such kernels in
// flight from two streams hung an earlier build of this library, and the cause was never isolated.  Each pair launch on a
// new stream first waits (cudaStreamWaitEvent) for the last pair launch of any other stream; same-stream launches are
// already ordered and pay nothing, and at the sizes where pair kernels are chosen each one fills the GPU on its own.
// Process-wide and thread-safe: the mutex is held across wait + launch + record.
std::mutex g_pair_mu;
cudaEvent_t g_pair_evt[MAX_DEV];
cudaStream_t g_pair_last_stream[MAX_DEV];
bool g_pair_evt_valid[MAX_DEV];
void pair_guard_begin(int dev, cudaStream_t st) {  // g_pair_mu held
  if (!g_pair_evt[dev] && cudaEventCreateWithFlags(&g_pair_evt[dev], cudaEventDisableTiming) != cudaSuccess) {
    g_pair_evt[dev] = nullptr;
    return;
  }
  if (g_pair_evt_valid[dev] && g_pair_last_stream[dev] != st) cudaStreamWaitEvent(st, g_pair_evt[dev], 0);
}
void pair_guard_end(int dev, cudaStream_t st) {  // g_pair_mu held
  if (!g_pair_evt[dev]) return;
  g_pair_evt_valid[dev] = cudaEventRecord(g_pair_evt[dev], st) == cudaSuccess;
  g_pair_last_stream[dev] = st;
}

template <int BN, int CL, int MODE, bool REUSE, int PASSES>
int launch_m(Ctx& ctx, const GemmTC& p, TCParams tp, int num_sms) {
  using KCfg = Cfg<BN, REUSE>;
  static std::atomic<bool> configured[MAX_DEV];
  if (configure_once(conv_gemm_wg_kernel<BN, CL, MODE, REUSE, PASSES>, configured, KCfg::SMEM)) return -2;
  static std::atomic<long long>* const counter = [] {
    static char name[48];
    const char* sp = PASSES == 1 ? ",fp16" : "";
    if (CL > 1) snprintf(name, sizeof(name), "tc2%s<%d,%s%s>", REUSE ? "r" : "", BN / 2, mode_name(MODE), sp);
    else snprintf(name, sizeof(name), "tc%s<%d,%s%s>", REUSE ? "r" : "", BN, mode_name(MODE), sp);
    return variant_counter(name);
  }();
  const ConvTC& w = *p.w;
  const int bi = map_index(BN / CL);
  const uint32_t a_rows = REUSE ? A3_ROWS : BM;  // REUSE: halo-extended activation boxes
  CUtensorMap ta_hi, ta_lo;
  if (cached_act_map(&ta_hi, p.A_hi, (uint64_t)p.rows_total, (uint64_t)w.Cin, a_rows)) return -1;
  if (PASSES == 1) ta_lo = ta_hi;  // never loaded
  else if (cached_act_map(&ta_lo, p.A_lo, (uint64_t)p.rows_total, (uint64_t)w.Cin, a_rows)) return -1;
  tp.NT = w.N / BN;
  const int total = (CL > 1 ? (tp.ntiles + 1) / 2 : tp.ntiles) * tp.NT;
  const int slots = num_sms / CL;
  const int ncl = total < slots ? total : slots;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(CL * ncl));
  cfg.blockDim = dim3(NTHREADS);
  cfg.dynamicSmemBytes = KCfg::SMEM;
  cfg.stream = ctx.stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;  // CL == 2: the two CTAs of a pair share a cluster (multicast, mapa)
  at[0].val.clusterDim.x = (unsigned)CL; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  {
    const bool guard = CL > 1;
    const int dev = guard ? current_device() : 0;
    std::unique_lock<std::mutex> lk(g_pair_mu, std::defer_lock);
    if (guard) {
      lk.lock();
      pair_guard_begin(dev, ctx.stream);
    }
    const cudaError_t le =
        cudaLaunchKernelEx(&cfg, conv_gemm_wg_kernel<BN, CL, MODE, REUSE, PASSES>, ta_hi, ta_lo, w.tm_hi[bi], w.tm_lo[bi], tp);
    if (guard) pair_guard_end(dev, ctx.stream);
    SSB_CUDA(le);
  }
  ++g_launches;
  counter->fetch_add(1, std::memory_order_relaxed);
  return 0;
}
template <int BN, int CL, int PASSES>
int launch(Ctx& ctx, const GemmTC& p, const TCParams& tp, int num_sms) {
  switch (tp.e.mode) {
    case EPI_GATE: return launch_m<BN, CL, EPI_GATE, false, PASSES>(ctx, p, tp, num_sms);
    case EPI_RES_SKIP: return launch_m<BN, CL, EPI_RES_SKIP, false, PASSES>(ctx, p, tp, num_sms);
    default: return launch_m<BN, CL, EPI_GENERIC, false, PASSES>(ctx, p, tp, num_sms);
  }
}
// the tap-reuse variant serves the CTA-pair sizes of 3-tap convs: the gate GEMMs of both denoisers, the vocoder's transposed
// convs (3-tap, N = u * C) and its k = 3 ResBlock convs
bool tap_reuse_eligible(const GemmTC& p, const ConvTC& w) {
  return w.taps == 3 && w.center == 1 && w.dil >= 1 && w.dil <= HALO && (p.e.mode == EPI_GATE || p.e.mode == EPI_GENERIC);
}
// large problems: CTA pairs (two row tiles x one 2*hb-wide N tile per cluster, the weight tile multicast to both) halve
// the weight bytes each SM pulls through L2
template <int PASSES>
int dispatch(Ctx& ctx, const GemmTC& p, const TCParams& tp, int num_sms) {
  const ConvTC& w = *p.w;
  if ((int64_t)((p.ntiles + 1) / 2) * (w.N / (2 * w.hb)) >= (int64_t)num_sms) {
    if (tap_reuse_eligible(p, w)) {
      if (p.e.mode == EPI_GATE)
        return w.hb == 64 ? launch_m<128, 2, EPI_GATE, true, PASSES>(ctx, p, tp, num_sms)
                          : launch_m<64, 2, EPI_GATE, true, PASSES>(ctx, p, tp, num_sms);
      return w.hb == 64 ? launch_m<128, 2, EPI_GENERIC, true, PASSES>(ctx, p, tp, num_sms)
                        : launch_m<64, 2, EPI_GENERIC, true, PASSES>(ctx, p, tp, num_sms);
    }
    return w.hb == 64 ? launch<128, 2, PASSES>(ctx, p, tp, num_sms) : launch<64, 2, PASSES>(ctx, p, tp, num_sms);
  }
  // smaller problems: single CTAs on 64-wide N tiles.  (A 128-wide single-CTA tile would need ntiles * N / 128 >= 2 #SMs,
  // which already meets the pair condition above when N % 128 == 0: it is never reached, so it is not built.)
  return launch<64, 1, PASSES>(ctx, p, tp, num_sms);
}

}  // namespace

bool tc_available() { return get_encode() != nullptr; }
int make_act_map(CUtensorMap* m, const void* ptr, int64_t rows, int cols, int box_rows) {
  return cached_act_map(m, ptr, (uint64_t)rows, (uint64_t)cols, (uint32_t)box_rows);
}
long long variant_launch_count(const char* name) {
  const int n = g_nvariants.load();
  for (int i = 0; i < n; ++i)
    if (strcmp(g_variants[i].name, name) == 0) return g_variants[i].n.load();
  return 0;
}
int variant_names(char* buf, int cap) {  // ';'-separated list of the variants launched so far
  int o = 0;
  const int n = g_nvariants.load();
  for (int i = 0; i < n; ++i) {
    const int l = (int)strlen(g_variants[i].name);
    if (o + l + 2 > cap) break;
    memcpy(buf + o, g_variants[i].name, l);
    o += l;
    buf[o++] = ';';
  }
  if (cap > 0) buf[o < cap ? o : cap - 1] = 0;
  return n;
}
void tensor_map_cache_stats(long long* encodes, long long* hits) {
  std::lock_guard<std::mutex> lk(g_host_mu);
  *encodes = g_map_encodes;
  *hits = g_map_hits;
}

int make_weight_maps(ConvTC* w) {
  SSB_CHECK(w->Cin % BK == 0 && w->N % 64 == 0, "tensor-core path needs Cin % 64 == 0 and N % 64 == 0");
  if (make_map(&w->tm_hi[0], w->W_hi, (uint64_t)w->taps * w->N, (uint64_t)w->Cin, 64)) return -1;
  if (make_map(&w->tm_lo[0], w->W_lo, (uint64_t)w->taps * w->N, (uint64_t)w->Cin, 64)) return -1;
  if (make_map(&w->tm_hi[1], w->W_hi, (uint64_t)w->taps * w->N, (uint64_t)w->Cin, 32)) return -1;
  if (make_map(&w->tm_lo[1], w->W_lo, (uint64_t)w->taps * w->N, (uint64_t)w->Cin, 32)) return -1;
  // CTA-pair kernel: each CTA of the pair loads hb weight rows of a 2*hb-wide N tile
  w->hb = w->N % 128 == 0 ? 64 : 32;
  w->ok = true;
  return 0;
}

int conv_gemm_tc(Ctx& ctx, const GemmTC& p) {
  if (ctx.dry || p.ntiles == 0) return 0;
  const ConvTC& w = *p.w;
  SSB_CHECK(w.ok, "conv_gemm_tc: weights not packed for the tensor-core path");
  SSB_CHECK(p.e.act == ACT_NONE || p.e.act == ACT_RELU || p.e.act == ACT_LRELU || p.e.act == ACT_GELU,
            "conv_gemm_tc: unsupported epilogue activation");
  SSB_CHECK(p.e.plane_act == ACT_NONE || p.e.plane_act == ACT_LRELU, "conv_gemm_tc: unsupported plane activation");
  SSB_CHECK(p.e.mode != EPI_GENERIC || p.e.out || p.e.oh, "conv_gemm_tc: GENERIC epilogue without an output");
  SSB_CHECK(p.e.mode != EPI_RES_SKIP || p.e.res || (p.e.rh && p.e.rl), "conv_gemm_tc: RES_SKIP epilogue without a residual source");
  const int num_sms = device_sms();
  TCParams tp;
  tp.tiles = p.tiles; tp.ntiles = p.ntiles; tp.taps = w.taps; tp.kchunks = w.Cin / BK;
  tp.dil = w.dil; tp.center = w.center; tp.N = w.N; tp.wscale = w.wscale; tp.e = p.e;
  if (!tp.e.bias) tp.e.bias = w.bias;
  return p.single_pass ? dispatch<1>(ctx, p, tp, num_sms) : dispatch<3>(ctx, p, tp, num_sms);
}

int split_planes(Ctx& ctx, const float* x, int ld, int64_t rows, int C, float scale, __half* hi, __half* lo) {
  if (ctx.dry || rows == 0) return 0;
  const int64_t n = rows * C;
  k_split_planes<<<(unsigned)((n + 255) / 256), 256, 0, ctx.stream>>>(x, ld, rows, C, scale, hi, lo);
  SSB_CUDA(cudaGetLastError());
  ++g_launches;
  return 0;
}

}  // namespace ssb
