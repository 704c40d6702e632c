// Multi-head attention (2 heads x 128) on Hopper tensor cores (wgmma) with TMA-staged tiles.  sm_90a only.
// Rows a3 / a12 of SURVEY.md section 8: self-attention of the FFT blocks (reference modules/commons/common_layers.py:277-286
// -> F.multi_head_attention_forward: q * hd^-0.5, bmm, key-padding -> -inf, fp32 softmax, bmm) and the style aligner's
// cross-attention (modules/StyleSinger/lse.py:41).  Used for long batches; short ones keep the fp32 kernel (attention.cu).
//
// One CTA = 128 queries of one (utterance, head); keys / values stream through a 4-slot shared-memory ring in tiles of 64.
// Both contractions are 3-pass fp16 hi/lo split MMAs like every other tensor-core GEMM of this library (fp32-class accuracy):
//   S   = Q K^T      M128 x N64  x K128 (head dim),  A = Q planes, B = K planes             -> registers
//   O  += P V        M128 x N128 x K64  (keys),      A = P planes from registers,           B = V^T planes -> registers
// No running rescale of O: pass 1 streams S once for the exact row maximum m, pass 2 recomputes S, forms
// p = exp(scale * (s - m)) (masked keys -> 0), accumulates l = sum p in registers and O += P V on the tensor cores; the
// epilogue divides by l.  P is carried as fp16 hi/lo planes of 256 * p so that weights down to 2^-33 survive the split.
// The [L, S] score matrix is never materialised (63 MB / utterance / layer in the reference at F = 2812).
//   warp 0: TMA producer   warps 4-11: two consumer warpgroups of 64 query rows each (MMAs, softmax, epilogue)
#include <stdlib.h>

#include <atomic>
#include <mutex>

#include "attention.cuh"
#include "conv_gemm_tc.cuh"
#include "tc_common.cuh"

namespace ssb {

namespace {

using namespace tc;

constexpr int AQ = 128, AK = 64, HD = 128;
constexpr int QT = AQ * 64 * 2;            // one [128 x 64] fp16 tile: 16 KB
constexpr int Q_BYTES = 4 * QT;            // hi_h0, hi_h1, lo_h0, lo_h1
constexpr int KT = AK * 64 * 2;            // one [64 keys x 64 d] fp16 tile: 8 KB
constexpr int SLOT = 4 * KT;               // K: hi_h0, hi_h1, lo_h0, lo_h1 ; V^T: hi [128 d x 64 keys], lo
constexpr int NSLOT = 4;
constexpr int ATT_THREADS = 384;
constexpr int ATT_SMEM = Q_BYTES + NSLOT * SLOT + 1024 + 256;
static_assert(ATT_SMEM <= 227 * 1024, "exceeds the 227 KB of shared memory a Hopper block can have");

struct AttnTCParams {
  const int4* utt_q;
  const int4* utt_k;
  int qcol0, kcol0;
  const float* keymask;
  float c2;  // scale * log2(e)
  float* out; int ldo;
  __half* oh; __half* ol; int ldh;
};

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tmQ_hi, const __grid_constant__ CUtensorMap tmQ_lo,
                    const __grid_constant__ CUtensorMap tmK_hi, const __grid_constant__ CUtensorMap tmK_lo,
                    const __grid_constant__ CUtensorMap tmV_hi, const __grid_constant__ CUtensorMap tmV_lo, const AttnTCParams p) {
  const int b = blockIdx.z, head = blockIdx.y;
  const int4 uq = p.utt_q[b], uk = p.utt_k[b];
  const int q0 = blockIdx.x * AQ;
  if (q0 >= uq.y) return;  // whole CTA, before any barrier state exists
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Q_BYTES + NSLOT * SLOT);  // qfull, kvfull[4], kvempty[4]
  const uint32_t qbase = smem_u32(smem), ring = qbase + Q_BYTES;
  const uint32_t qfull = smem_u32(bars), kvfull0 = qfull + 8, kvempty0 = kvfull0 + 8 * NSLOT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    mbar_init(qfull, 1);
    for (int s = 0; s < NSLOT; ++s) {
      mbar_init(kvfull0 + 8 * s, 1);
      mbar_init(kvempty0 + 8 * s, 8);  // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // Key tiles sit on a grid aligned to 8 rows of the K/V layout: the V^T planes are read with the key index as the INNER
  // TMA coordinate, whose byte offset must be a multiple of 16.  The (up to 7) rows in front of the utterance are masked.
  const int klen = uk.y;
  const int kshift = uk.x & 7;
  const int krow0 = uk.x - kshift;
  const int n = (kshift + klen + AK - 1) / AK;  // key tiles
  const int qrow0 = uq.x + q0;
  const int hq = p.qcol0 + head * HD, hk = p.kcol0 + head * HD;

  if (warp == 0) {
    if (lane == 0) {
      mbar_expect_tx(qfull, Q_BYTES);
      tma_load_2d(qbase, &tmQ_hi, qfull, hq, qrow0);
      tma_load_2d(qbase + QT, &tmQ_hi, qfull, hq + 64, qrow0);
      tma_load_2d(qbase + 2 * QT, &tmQ_lo, qfull, hq, qrow0);
      tma_load_2d(qbase + 3 * QT, &tmQ_lo, qfull, hq + 64, qrow0);
      int slot = 0;
      uint32_t ph = 0;
      auto load_k = [&](int j) {
        mbar_wait(kvempty0 + 8 * slot, ph ^ 1);
        const uint32_t fb = kvfull0 + 8 * slot, sa = ring + slot * SLOT;
        mbar_expect_tx(fb, SLOT);
        tma_load_2d(sa, &tmK_hi, fb, hk, krow0 + j * AK);
        tma_load_2d(sa + KT, &tmK_hi, fb, hk + 64, krow0 + j * AK);
        tma_load_2d(sa + 2 * KT, &tmK_lo, fb, hk, krow0 + j * AK);
        tma_load_2d(sa + 3 * KT, &tmK_lo, fb, hk + 64, krow0 + j * AK);
        if (++slot == NSLOT) { slot = 0; ph ^= 1; }
      };
      auto load_v = [&](int j) {  // V^T planes [heads * 128, key rows]: box = 64 keys x 128 d
        mbar_wait(kvempty0 + 8 * slot, ph ^ 1);
        const uint32_t fb = kvfull0 + 8 * slot, sa = ring + slot * SLOT;
        mbar_expect_tx(fb, SLOT);
        tma_load_2d(sa, &tmV_hi, fb, krow0 + j * AK, head * HD);
        tma_load_2d(sa + 2 * KT, &tmV_lo, fb, krow0 + j * AK, head * HD);
        if (++slot == NSLOT) { slot = 0; ph ^= 1; }
      };
      for (int j = 0; j < n; ++j) load_k(j);  // pass 1: row maxima
      for (int j = 0; j < n; ++j) {           // pass 2, in the order the consumers use them: K0, V0, K1, V1, ...
        load_k(j);
        load_v(j);
      }
    }
  } else if (warp >= 4) {
    // consumer warpgroup cw: query rows [64 cw, 64 cw + 64) of the tile; this thread holds rows rw and rw + 8 of them
    const int cw = (warp - 4) >> 2, wq = warp & 3;
    const int rw = 16 * wq + (lane >> 2);
    const uint32_t qoff = (uint32_t)cw * 8192u;
    int slot = 0;
    uint32_t ph = 0;
    auto release = [&]() {
      __syncwarp();
      if (lane == 0) mbar_arrive(kvempty0 + 8 * slot);
      if (++slot == NSLOT) { slot = 0; ph ^= 1; }
    };
    // S = Q K^T for the key tile in the current slot (3-pass split), then the slot goes back to the producer
    float s[32];
    auto scores = [&]() {
      mbar_wait(kvfull0 + 8 * slot, ph);
      const uint32_t sa = ring + slot * SLOT;
      wg_fence();
      fence_acc(s);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint64_t off = (uint64_t)((ks * 32) >> 4);
          const uint64_t qh = make_sdesc(qbase + h * QT + qoff) + off, ql = make_sdesc(qbase + 2 * QT + h * QT + qoff) + off;
          const uint64_t kh = make_sdesc(sa + h * KT) + off, kl = make_sdesc(sa + 2 * KT + h * KT) + off;
          wgmma_n64(s, qh, kh, (h | ks) != 0 ? 1u : 0u);
          wgmma_n64(s, qh, kl, 1u);
          wgmma_n64(s, ql, kh, 1u);
        }
      }
      wg_commit();
      fence_acc(s);
      wg_wait<0>();
      fence_acc(s);
      release();
    };
    // valid keys among this thread's 16 columns of key tile j: bit j of the mask <-> accumulator element j / j + 2
    auto key_mask = [&](int j) {
      uint32_t m = 0;
#pragma unroll
      for (int e = 0; e < 16; ++e) {
        const int c = frag_col(lane, (e >> 1) * 4 + (e & 1));
        const int k = j * AK + c - kshift;  // key index inside the utterance
        bool v = k >= 0 && k < klen;
        if (v && p.keymask) v = __ldg(p.keymask + uk.x + k) != 0.f;
        m |= (v ? 1u : 0u) << e;
      }
      return m;
    };
    mbar_wait(qfull, 0);
    // pass 1: exact row maximum of the raw scores over the valid keys
    float m0 = -INFINITY, m1 = -INFINITY;
    for (int j = 0; j < n; ++j) {
      const uint32_t km = key_mask(j);
      scores();
#pragma unroll
      for (int e = 0; e < 16; ++e) {
        if ((km >> e) & 1u) {
          const int jj = (e >> 1) * 4 + (e & 1);
          m0 = fmaxf(m0, s[jj]);
          m1 = fmaxf(m1, s[jj + 2]);
        }
      }
    }
#pragma unroll
    for (int x = 1; x <= 2; x <<= 1) {
      m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, x));
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, x));
    }
    const float mu0 = m0 == -INFINITY ? 0.f : m0, mu1 = m1 == -INFINITY ? 0.f : m1;
    const float c2 = p.c2;
    float l0 = 0.f, l1 = 0.f;
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;
    // pass 2: p = exp(scale * (s - m)); O += P V with P as the register A operand (fp16 hi/lo planes of 256 p, so that
    // weights down to 2^-33 survive the split)
    for (int j = 0; j < n; ++j) {
      const uint32_t km = key_mask(j);
      scores();
      float pv[32];
#pragma unroll
      for (int e = 0; e < 16; ++e) {
        const int jj = (e >> 1) * 4 + (e & 1);
        const bool v = (km >> e) & 1u;
        pv[jj] = v ? exp2f((s[jj] - mu0) * c2) : 0.f;
        pv[jj + 2] = v ? exp2f((s[jj + 2] - mu1) * c2) : 0.f;
        l0 += pv[jj];
        l1 += pv[jj + 2];
      }
      uint32_t ah[4][4], al[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float x0 = pv[8 * kk + 2 * q] * 256.0f, x1 = pv[8 * kk + 2 * q + 1] * 256.0f;
          const __half2 hh = __floats2half2_rn(x0, x1);
          const float2 hf = __half22float2(hh);
          ah[kk][q] = *reinterpret_cast<const uint32_t*>(&hh);
          al[kk][q] = pack_half2(x0 - hf.x, x1 - hf.y);
        }
      }
      mbar_wait(kvfull0 + 8 * slot, ph);
      const uint32_t sv = ring + slot * SLOT;
      wg_fence();
      fence_acc(o);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint64_t off = (uint64_t)((kk * 32) >> 4);
        const uint64_t vh = make_sdesc(sv) + off, vl = make_sdesc(sv + 2 * KT) + off;
        wgmma_rs_n128(o, ah[kk], vh, 1u);
        wgmma_rs_n128(o, ah[kk], vl, 1u);
        wgmma_rs_n128(o, al[kk], vh, 1u);
      }
      wg_commit();
      fence_acc(o);
      wg_wait<0>();
      fence_acc(o);
      release();
    }
#pragma unroll
    for (int x = 1; x <= 2; x <<= 1) {
      l0 += __shfl_xor_sync(0xffffffffu, l0, x);
      l1 += __shfl_xor_sync(0xffffffffu, l1, x);
    }
    // epilogue: O / (256 l).  l >= 1 when any key is valid (the maximum contributes exp2(0)); a row without one has l = 0 and
    // O = 0 and writes 0 * inf = NaN, like the fp32 kernel and torch's softmax over all -inf
    const float inv0 = 1.0f / (256.0f * l0), inv1 = 1.0f / (256.0f * l1);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int qr = 64 * cw + rw + 8 * hh;  // query row inside the tile
      if (q0 + qr >= uq.y) continue;
      const int64_t grow = (int64_t)qrow0 + qr;
      const float inv = hh ? inv1 : inv0;
#pragma unroll
      for (int nb = 0; nb < 16; ++nb) {
        const int jj = 4 * nb + 2 * hh;
        const int col = head * HD + frag_col(lane, jj);
        const float a = o[jj] * inv, bb = o[jj + 1] * inv;
        if (p.out) *reinterpret_cast<float2*>(p.out + grow * p.ldo + col) = make_float2(a, bb);
        if (p.oh) {
          const __half2 h2 = __floats2half2_rn(a, bb);
          const float2 hf = __half22float2(h2);
          *reinterpret_cast<__half2*>(p.oh + grow * p.ldh + col) = h2;
          *reinterpret_cast<__half2*>(p.ol + grow * p.ldh + col) = __floats2half2_rn(a - hf.x, bb - hf.y);
        }
      }
    }
  }
}

// planes [rows, ld] (columns col0 .. col0 + C) -> transposed planes [C, ldt] (ldt >= rows)
__global__ void k_transpose_planes(const __half* __restrict__ xh, const __half* __restrict__ xl, int ld, int col0, int64_t rows,
                                   __half* __restrict__ th, __half* __restrict__ tl, int64_t ldt) {
  __shared__ __half sh[32][34], sl[32][34];
  const int64_t r0 = (int64_t)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 256 threads: ty 0..7
  for (int i = ty; i < 32; i += 8) {
    const int64_t r = r0 + i;
    sh[i][tx] = r < rows ? xh[r * ld + col0 + c0 + tx] : __float2half(0.f);
    sl[i][tx] = r < rows ? xl[r * ld + col0 + c0 + tx] : __float2half(0.f);
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int64_t r = r0 + tx;
    if (r < ldt) {
      th[(int64_t)(c0 + i) * ldt + r] = sh[tx][i];
      tl[(int64_t)(c0 + i) * ldt + r] = sl[tx][i];
    }
  }
}

}  // namespace

static std::atomic<int> g_attn_tc{1};  // default on (checked against the fp32 kernel by tests/test_gpu_tc.py)
bool attention_tc_enabled() { return g_attn_tc.load(std::memory_order_relaxed) != 0 && tc_available(); }
int set_attention_tc_enabled(int on) {
  g_attn_tc.store(on ? 1 : 0, std::memory_order_relaxed);
  return on ? 1 : 0;
}

int transpose_planes(Ctx& ctx, const __half* xh, const __half* xl, int ld, int col0, int64_t rows, int C, __half* th, __half* tl,
                     int64_t ldt) {
  SSB_CHECK(C % 32 == 0 && ldt >= rows && col0 >= 0 && col0 + C <= ld, "transpose_planes: bad shape");
  if (ctx.dry || rows == 0) return 0;
  dim3 grid((unsigned)((ldt + 31) / 32), (unsigned)(C / 32));
  k_transpose_planes<<<grid, 256, 0, ctx.stream>>>(xh, xl, ld, col0, rows, th, tl, ldt);
  SSB_CUDA(cudaGetLastError());
  ++g_launches;
  return 0;
}

int attention_tc_check(const AttnTCArgs& a) {
  SSB_CHECK(a.heads == 1 || a.heads == 2, "attention_tc: heads must be 1 or 2, got " + std::to_string(a.heads));
  SSB_CHECK(a.B >= 0 && a.B <= 65535, "attention_tc: B = " + std::to_string(a.B) + " exceeds gridDim.z (65535)");
  SSB_CHECK(a.out || (a.oh && a.ol), "attention_tc: no output");
  SSB_CHECK(a.ldq % 8 == 0 && a.ldk % 8 == 0 && a.ldvt % 8 == 0 && a.ldo % 8 == 0 && a.ldh % 8 == 0,
            "attention_tc: ldq / ldk / ldvt / ldo / ldh must be multiples of 8");
  SSB_CHECK(a.qcol0 >= 0 && a.kcol0 >= 0 && a.qcol0 % 8 == 0 && a.kcol0 % 8 == 0,
            "attention_tc: qcol0 / kcol0 must be non-negative multiples of 8 (TMA inner coordinates)");
  SSB_CHECK(((uintptr_t)a.Qh | (uintptr_t)a.Ql | (uintptr_t)a.Kh | (uintptr_t)a.Kl | (uintptr_t)a.Vth | (uintptr_t)a.Vtl |
             (uintptr_t)a.out | (uintptr_t)a.oh | (uintptr_t)a.ol) % 16 == 0,
            "attention_tc: every operand and output must be 16-byte aligned");
  const int w = a.heads * HD;
  SSB_CHECK(a.qcol0 + w <= a.ldq, "attention_tc: Q columns qcol0 + heads x 128 = " + std::to_string(a.qcol0 + w) +
                                      " exceed ldq = " + std::to_string(a.ldq));
  SSB_CHECK(a.kcol0 + w <= a.ldk, "attention_tc: K columns kcol0 + heads x 128 = " + std::to_string(a.kcol0 + w) +
                                      " exceed ldk = " + std::to_string(a.ldk));
  SSB_CHECK((!a.out || a.ldo >= w) && (!a.oh || a.ldh >= w), "attention_tc: an output ld is narrower than heads x 128");
  SSB_CHECK(a.ldvt >= a.rows_k, "attention_tc: ldvt is smaller than the key rows");
  return 0;
}

int attention_tc(Ctx& ctx, const AttnTCArgs& a) {
  if (attention_tc_check(a)) return -1;
  if (ctx.dry || a.B == 0 || a.max_q == 0) return 0;
  {
    static std::atomic<bool> configured[64];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!configured[dev].load(std::memory_order_acquire)) {
      SSB_CUDA(cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM));
      configured[dev].store(true, std::memory_order_release);
    }
  }
  CUtensorMap mq_h, mq_l, mk_h, mk_l, mv_h, mv_l;
  if (make_act_map(&mq_h, a.Qh, a.rows_q, a.ldq, AQ)) return -1;
  if (make_act_map(&mq_l, a.Ql, a.rows_q, a.ldq, AQ)) return -1;
  if (make_act_map(&mk_h, a.Kh, a.rows_k, a.ldk, AK)) return -1;
  if (make_act_map(&mk_l, a.Kl, a.rows_k, a.ldk, AK)) return -1;
  if (make_act_map(&mv_h, a.Vth, (int64_t)a.heads * HD, (int)a.ldvt, HD)) return -1;
  if (make_act_map(&mv_l, a.Vtl, (int64_t)a.heads * HD, (int)a.ldvt, HD)) return -1;
  AttnTCParams p;
  p.utt_q = a.utt_q; p.utt_k = a.utt_k; p.qcol0 = a.qcol0; p.kcol0 = a.kcol0; p.keymask = a.keymask;
  p.c2 = a.scale * 1.4426950408889634f;
  p.out = a.out; p.ldo = a.ldo; p.oh = a.oh; p.ol = a.ol; p.ldh = a.ldh;
  dim3 grid((a.max_q + AQ - 1) / AQ, a.heads, a.B);
  attention_tc_kernel<<<grid, ATT_THREADS, ATT_SMEM, ctx.stream>>>(mq_h, mq_l, mk_h, mk_l, mv_h, mv_l, p);
  SSB_CUDA(cudaGetLastError());
  ++g_launches;
  ++g_attn_launches[1];
  return 0;
}

}  // namespace ssb
