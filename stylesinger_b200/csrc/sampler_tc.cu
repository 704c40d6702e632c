// Persistent mel-diffusion sampler: ONE cooperative kernel launch runs all T reverse steps
// (DiffusionDecoder.forward(infer=True), reference modules/diff/shallow_diffusion_tts.py:284-307, over
// DiffNet, modules/diff/net.py:107-130) for a (small) ragged batch.  BASELINE.json north_star: "the T-step
// diffusion loop fused into a persistent kernel that keeps the mel state resident and launches once per
// utterance"; configs[4] compares it with the per-step-launch path (ssb_model_set_persistent).
//
// Structure: a 64-wide conv GEMM (TMA -> 4-stage smem ring -> 3-pass fp16 split wgmma into register accumulators ->
// shared-memory staging -> per-row fused epilogue) wrapped in a loop over a PHASE TABLE in device memory:
//   per step t:  in_proj | 20 x (dilated conv + conditioner -> gate ; 1x1 -> residual/skip) | skip_proj |
//                out_proj + DDPM posterior update (q_posterior + noise) writing x_{t-1} and its fp16 planes
// = 43 GEMM phases per step, separated by a grid-wide barrier (every phase reads what all CTAs wrote in
// the previous one through +-dilation halos).  Tensor maps (activations + every layer's weights) live in a
// device array; mbarrier phases and the smem ring persist across all 43*T phases.
// PASSES = 1 (single-pass fp16, the mel sampler under ssb_model_set_mel_precision(SSB_TC_FP16)): only the hi planes of A and
// W are loaded and each K step issues one wgmma per accumulator; the stage layout stays that of PASSES = 3.
#include <cuda_fp16.h>
#include <string.h>

#include "philox.cuh"
#include <mutex>

#include "sampler_tc.cuh"
#include "tc_common.cuh"

namespace ssb {

namespace {

using namespace tc;

constexpr int BM = 128, BK = 64, BN = 64;
constexpr int A_TILE = BM * BK * 2;     // 16 KB
constexpr int B_TILE = BN * BK * 2;     // 8 KB
constexpr int STAGE = 2 * A_TILE + 2 * B_TILE;  // 48 KB
constexpr int STAGES = 4;
constexpr int ACC_BYTES = BM * BN * 4;     // accumulator staging [128 rows x 64] fp32, float4 chunks XOR-swizzled by row
constexpr int SMEM = STAGES * STAGE + ACC_BYTES + 1024 + 512 + 1024;
static_assert(SMEM <= 227 * 1024, "exceeds the 227 KB of shared memory a Hopper block can have");
static_assert(sizeof(SPhase) <= 1024, "the phase descriptor is staged in a 1 KB shared-memory slot");

__device__ __forceinline__ void proxy_fence() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ uint32_t cluster_id_x() { uint32_t r; asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t ncluster_id_x() { uint32_t r; asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r)); return r; }

__device__ __forceinline__ void grid_barrier(unsigned* ctr, unsigned& gen, unsigned nblocks) {
  __threadfence();
  proxy_fence();
  __syncthreads();
  if (threadIdx.x == 0) {
    ++gen;
    const unsigned target = gen * nblocks;
    __threadfence();
    atomicAdd(ctr, 1u);
    const long long t0 = clock64();
    while (true) {
      unsigned v;
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
      if (v >= target) break;
      if (clock64() - t0 > 8000000000LL) __trap();
    }
    __threadfence();
    proxy_fence();
  }
  __syncthreads();
}

struct Pre {
  float4 a[8];
};

__device__ __forceinline__ void prefetch32(const SPhase& e, int64_t r, int n, bool valid, Pre& p) {
  if (!valid) return;
  if (e.mode == SP_RES_SKIP) {
    if (n < e.C) {
      const float4* rp = reinterpret_cast<const float4*>(e.res + r * e.ld_res + n);
#pragma unroll
      for (int q = 0; q < 8; ++q) p.a[q] = __ldcg(rp + q);
    } else if (!e.skip_init) {
      const float4* sp = reinterpret_cast<const float4*>(e.skip + r * e.ld_skip + (n - e.C));
#pragma unroll
      for (int q = 0; q < 8; ++q) p.a[q] = __ldcg(sp + q);
    }
  } else if (e.mode == SP_GATE) {
    const float4* ap = reinterpret_cast<const float4*>(e.add + r * e.ld_add + n);
#pragma unroll
    for (int q = 0; q < 8; ++q) p.a[q] = __ldg(ap + q);
  } else if (e.mode == SP_MEL_SAMPLE) {
    const float4* xp = reinterpret_cast<const float4*>(e.out + r * e.ldo + n);
#pragma unroll
    for (int q = 0; q < 8; ++q)
      if (n + 4 * q < e.n_valid) p.a[q] = __ldcg(xp + q);
  }
}

// ti: the row's tight index in the call (injected noise); g, lr: its utterance's Philox entry and its row inside the
// utterance (Philox counter row g->row0 + lr)
__device__ __forceinline__ void epilogue32(const SPhase& e, int64_t r, int64_t ti, const UttRng* g, int lr, int n,
                                           const uint32_t (&raw)[32], const Pre& pre) {
  float v[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = fmaf(__uint_as_float(raw[j]), e.wscale, __ldg(e.bias + n + j));
  if (e.mode == SP_GATE) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      v[4 * q] += pre.a[q].x; v[4 * q + 1] += pre.a[q].y; v[4 * q + 2] += pre.a[q].z; v[4 * q + 3] += pre.a[q].w;
    }
    float z[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) z[q] = gate_act(v[2 * q], v[2 * q + 1]);
    split_store16(e.oh + r * e.ldh + (n >> 1), e.ol + r * e.ldh + (n >> 1), z);
    return;
  }
  if (e.mode == SP_RES_SKIP) {
    if (n < e.C) {
      float4* op = reinterpret_cast<float4*>(e.out + r * e.ldo + n);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 x0 = pre.a[q];
        v[4 * q] = (v[4 * q] + x0.x) * e.beta;
        v[4 * q + 1] = (v[4 * q + 1] + x0.y) * e.beta;
        v[4 * q + 2] = (v[4 * q + 2] + x0.z) * e.beta;
        v[4 * q + 3] = (v[4 * q + 3] + x0.w) * e.beta;
        op[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
      }
      if (e.oh) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] += __ldg(e.vec2 + n + j);
        split_store16(e.oh + r * e.ldh + n, e.ol + r * e.ldh + n, v);
        split_store16(e.oh + r * e.ldh + n + 16, e.ol + r * e.ldh + n + 16, v + 16);
      }
    } else {
      const int sc = n - e.C;
      float4* sp = reinterpret_cast<float4*>(e.skip + r * e.ld_skip + sc);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        if (!e.skip_init) {
          const float4 o = pre.a[q];
          v[4 * q] += o.x; v[4 * q + 1] += o.y; v[4 * q + 2] += o.z; v[4 * q + 3] += o.w;
        }
        sp[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
      }
      if (e.sh) {  // last layer: the finished skip sum also goes out as fp16 planes (A operand of skip_proj)
        split_store16(e.sh + r * e.C + sc, e.sl + r * e.C + sc, v);
        split_store16(e.sh + r * e.C + sc + 16, e.sl + r * e.C + sc + 16, v + 16);
      }
    }
    return;
  }
  if (e.mode == SP_F0_SAMPLE) {
    if (n != 0) return;  // columns 0..2 of the (padded) 3-channel head: (eps, logit0, logit1)
    const float ln2 = 0.69314718055994530942f;
    const float zt = __ldcg(e.out + r);
    float x0 = __ldg(e.tab + 0) * zt - __ldg(e.tab + 1) * v[0];
    x0 = fmaxf(fminf(x0, __ldg(e.clip_hi + r)), __ldg(e.clip_lo + r));
    const float mean = __ldg(e.tab + 2) * x0 + __ldg(e.tab + 3) * zt;
    const float gz = e.noise ? __ldg(e.noise + ti) : philox_normal(g->key, e.stream_id, (uint64_t)((int64_t)g->row0 + lr));
    const float zn = mean + __ldg(e.tab + 4) * gz;
    e.out[r] = zn;
    const float l0a = v[1], l0b = v[2];
    const float mx = fmaxf(l0a, l0b);
    const float lse = mx + logf(expf(l0a - mx) + expf(l0b - mx));
    const float ls0 = l0a - lse, ls1 = l0b - lse;
    auto lae = [](float a, float b) { const float m = fmaxf(a, b); return m + logf(expf(a - m) + expf(b - m)); };
    float e0, e1;
    if (e.tstep == 0) { e0 = ls0; e1 = ls1; }
    else {
      e0 = lae(ls0 + __ldg(e.tab2 + 2), __ldg(e.tab2 + 3) - ln2);
      e1 = lae(ls1 + __ldg(e.tab2 + 2), __ldg(e.tab2 + 3) - ln2);
    }
    const int cur = e.uv[r];
    const float lz0 = cur == 0 ? 0.f : e.log_eps, lz1 = cur == 1 ? 0.f : e.log_eps;
    const float u0 = e0 + lae(lz0 + __ldg(e.tab2 + 0), __ldg(e.tab2 + 1) - ln2);
    const float u1 = e1 + lae(lz1 + __ldg(e.tab2 + 0), __ldg(e.tab2 + 1) - ln2);
    const float m2 = fmaxf(u0, u1);
    const float lse2 = m2 + logf(expf(u0 - m2) + expf(u1 - m2));
    const float p0 = u0 - lse2, p1 = u1 - lse2;
    const uint64_t gc = (uint64_t)((int64_t)g->row0 + lr) * 2;
    const float r0 = e.noise2 ? __ldg(e.noise2 + ti * 2) : philox_uniform(g->key, e.stream2, gc);
    const float r1 = e.noise2 ? __ldg(e.noise2 + ti * 2 + 1) : philox_uniform(g->key, e.stream2, gc + 1);
    const float g0 = -logf(-logf(r0 + 1e-30f) + 1e-30f);
    const float g1 = -logf(-logf(r1 + 1e-30f) + 1e-30f);
    const int cls = (g1 + p1) > (g0 + p0) ? 1 : 0;
    e.uv[r] = cls;
    if (e.has_next) {  // DDiffNet input of step t-1 (net.py:249-252): cat[Conv1x1(f0), Embedding(uv)] ; y = x + d0
      const int C = e.C, h = C / 2;
      for (int c0 = 0; c0 < C; c0 += 16) {
        float xv[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int c = c0 + j;
          xv[j] = c < h ? (zn * __ldg(e.in_w + c) + __ldg(e.in_b + c)) : __ldg(e.uv_emb + cls * h + (c - h));
        }
        float4* xp = reinterpret_cast<float4*>(e.x_next + r * C + c0);
#pragma unroll
        for (int q = 0; q < 4; ++q) xp[q] = make_float4(xv[4 * q], xv[4 * q + 1], xv[4 * q + 2], xv[4 * q + 3]);
#pragma unroll
        for (int j = 0; j < 16; ++j) xv[j] += __ldg(e.vec2 + c0 + j);
        split_store16(e.oh + r * e.ldh + c0, e.ol + r * e.ldh + c0, xv);
      }
    }
    return;
  }
  if (e.mode == SP_INPROJ || e.mode == SP_SKIPPROJ) {
    if (e.mode == SP_SKIPPROJ && e.n_valid > 0 && n >= e.n_valid) return;
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.0f);
    if (e.out) {
      float4* op = reinterpret_cast<float4*>(e.out + r * e.ldo + n);
#pragma unroll
      for (int q = 0; q < 8; ++q) op[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    }
    if (e.vec2) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] += __ldg(e.vec2 + n + j);
    }
    split_store16(e.oh + r * e.ldh + n, e.ol + r * e.ldh + n, v);
    split_store16(e.oh + r * e.ldh + n + 16, e.ol + r * e.ldh + n + 16, v + 16);
    return;
  }
  if (e.mode == SP_MEL_SAMPLE) {
    // p_sample (shallow_diffusion_tts.py:155-162): v = eps for columns n..n+31 (valid below n_valid).  ProDiff
    // (prodiff.py:143-148): v = x0 itself; its table holds (0, -1) in slots 0-1 and no_clip is set.
    if (n >= e.n_valid) return;
    const float a = __ldg(e.tab + 0), bq = __ldg(e.tab + 1), c1 = __ldg(e.tab + 2), c2 = __ldg(e.tab + 3), sig = __ldg(e.tab + 4);
    // clip bound 1 (DDPM) or +inf (ProDiff: no clip).  A bound rather than a branch keeps the kernel at its register count.
    const float lim = e.no_clip ? __int_as_float(0x7f800000) : 1.0f;
    float xn[32];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      if (n + 4 * q >= e.n_valid) {
        xn[4 * q] = xn[4 * q + 1] = xn[4 * q + 2] = xn[4 * q + 3] = 0.f;
        continue;
      }
      const float xs[4] = {pre.a[q].x, pre.a[q].y, pre.a[q].z, pre.a[q].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int c = n + 4 * q + k;
        const float xt = xs[k];
        float x0 = a * xt - bq * v[4 * q + k];
        x0 = fminf(fmaxf(x0, -lim), lim);
        const float mean = c1 * x0 + c2 * xt;
        const float nz = e.noise ? __ldg(e.noise + ti * 80 + c)
                                 : philox_normal(g->key, e.stream_id, (uint64_t)((int64_t)g->row0 + lr) * 80 + c);
        xn[4 * q + k] = mean + sig * nz;
      }
      *reinterpret_cast<float4*>(e.out + r * e.ldo + n + 4 * q) = make_float4(xn[4 * q], xn[4 * q + 1], xn[4 * q + 2], xn[4 * q + 3]);
    }
    // planes of x_{t-1} (padded to ldh columns; columns >= n_valid stay zero)
    if (n + 16 <= e.n_valid) split_store16(e.oh + r * e.ldh + n, e.ol + r * e.ldh + n, xn);
    if (n + 32 <= e.n_valid) split_store16(e.oh + r * e.ldh + n + 16, e.ol + r * e.ldh + n + 16, xn + 16);
    return;
  }
}

template <int PASSES>
__global__ void __launch_bounds__(256, 1)
sampler_tc_kernel(const CUtensorMap* __restrict__ maps, const SPhase* __restrict__ phases, int nphases,
                  const int2* __restrict__ tiles, const int4* __restrict__ tile_pos, const UttRng* __restrict__ rng,
                  int ntiles, unsigned* barrier_ctr, int cs) {
  // cs = cluster size along N: the cs CTAs of a cluster work on the same M-tile (consecutive N-tiles); each loads
  // 1/cs of the A tile and TMA-multicasts it to all of them, so the activation planes cross L2->SM once per
  // cluster instead of once per CTA.  Stage recycling therefore needs every CTA of the cluster to have consumed
  // the stage: each consumer warp arrives on the empty barrier of all cs CTAs (count 4 cs).
  // warp 0: TMA producer; warps 4-7: one consumer warpgroup (wgmma for rows 0-63 and 64-127, then the epilogue, thread =
  // row); warps 1-3 only take part in the phase-descriptor staging and the barriers.
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float4* accs = reinterpret_cast<float4*>(smem + STAGES * STAGE);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE + ACC_BYTES);
  SPhase* sph = reinterpret_cast<SPhase*>(smem + STAGES * STAGE + ACC_BYTES + 512);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t full0 = smem_u32(bars), empty0 = full0 + 8 * STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, (uint32_t)(4 * cs));
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int cr = cs > 1 ? (int)cluster_rank() : 0;
  const int cid = cs > 1 ? (int)cluster_id_x() : (int)blockIdx.x;
  const int ncl = cs > 1 ? (int)ncluster_id_x() : (int)gridDim.x;
  const uint16_t cmask = (uint16_t)((1u << cs) - 1u);
  const int slice_rows = BM / cs;
  const uint32_t slice_bytes = (uint32_t)(slice_rows * BK * 2);
  if (cs > 1) cluster_sync_all();  // every CTA's barriers are initialised before any remote arrive / multicast

  // pipeline state, persistent across phases (each role keeps its own copy)
  int stage = 0;
  uint32_t phase_bit = 0;
  unsigned gen = 0;

  for (int ph = 0; ph < nphases; ++ph) {
    // stage the phase descriptor in shared memory
    {
      const uint32_t* src = reinterpret_cast<const uint32_t*>(phases + ph);
      uint32_t* dst = reinterpret_cast<uint32_t*>(sph);
      for (int i = threadIdx.x; i < (int)(sizeof(SPhase) / 4); i += blockDim.x) dst[i] = __ldg(src + i);
    }
    __syncthreads();
    const SPhase& P = *sph;
    const int gpm = P.NT / cs;           // tile groups (clusters' worth of N-tiles) per M-tile
    const int groups = ntiles * gpm;
    const int g_first = ((cid - P.goff) % ncl + ncl) % ncl;  // group g runs on cluster (g + goff) % ncl
    const int nk = P.taps * P.kchunks;

    if (warp == 0) {
      if (lane == 0) {
        proxy_fence();
        const CUtensorMap* mA = maps + P.a1;
        const CUtensorMap* mW = maps + P.w1;
        for (int g = g_first; g < groups; g += ncl) {
          const int mt = g / gpm, nt = (g - mt * gpm) * cs + cr;
          const int row0 = tiles[mt].x;
          for (int kb = 0; kb < nk; ++kb) {
            mbar_wait(empty0 + 8 * stage, phase_bit ^ 1);
            const uint32_t fb = full0 + 8 * stage;
            mbar_expect_tx(fb, PASSES == 3 ? STAGE : A_TILE + B_TILE);
            const uint32_t sa = sbase + stage * STAGE;
            const int tap = kb / P.kchunks;
            const int c0 = (kb - tap * P.kchunks) * BK;
            const int arow = row0 + (tap - P.center) * P.dil;
            const int brow = tap * P.N + nt * BN;
            if (cs > 1) {
              tma_load_2d_mc(sa + cr * slice_bytes, mA, fb, c0, arow + cr * slice_rows, cmask);
              if constexpr (PASSES == 3) tma_load_2d_mc(sa + A_TILE + cr * slice_bytes, mA + 1, fb, c0, arow + cr * slice_rows, cmask);
            } else {
              tma_load_2d(sa, mA, fb, c0, arow);
              if constexpr (PASSES == 3) tma_load_2d(sa + A_TILE, mA + 1, fb, c0, arow);
            }
            tma_load_2d(sa + 2 * A_TILE, mW, fb, c0, brow);
            if constexpr (PASSES == 3) tma_load_2d(sa + 2 * A_TILE + B_TILE, mW + 1, fb, c0, brow);
            if (++stage == STAGES) { stage = 0; phase_bit ^= 1; }
          }
        }
      }
      __syncwarp();
    } else if (warp >= 4) {
      const int ew = warp - 4;
      auto release = [&](int st) {  // this warp is done reading stage st: tell every CTA that multicasts into it
        __syncwarp();
        if (lane == 0) {
          const uint32_t bar = empty0 + 8 * st;
          if (cs > 1) {
            for (int r = 0; r < cs; ++r) mbar_arrive_cluster(mapa_u32(bar, (uint32_t)r));
          } else {
            mbar_arrive(bar);
          }
        }
      };
      for (int g = g_first; g < groups; g += ncl) {
        const int mt = g / gpm, nt = (g - mt * gpm) * cs + cr;
        const int2 t = tiles[mt];
        const int rl = ew * 32 + lane;
        const bool valid = rl < t.y;
        const int64_t r = (int64_t)t.x + rl;
        const int4 tp = tile_pos[mt];  // tiles never straddle utterances
        const int64_t ti = (int64_t)tp.x + rl;
        const UttRng* ug = rng + tp.y;
        const int lr = tp.z + rl;
        Pre cur, nxt;
        prefetch32(P, r, nt * BN, valid, cur);
        float acc0[BN / 2], acc1[BN / 2];  // rows [0, 64) and [64, 128) of the tile
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc0[i] = acc1[i] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < nk; ++kb) {
          mbar_wait(full0 + 8 * stage, phase_bit);
          const uint32_t sa = sbase + stage * STAGE;
          const uint64_t dah = make_sdesc(sa), dal = make_sdesc(sa + A_TILE);
          const uint64_t dbh = make_sdesc(sa + 2 * A_TILE), dbl = make_sdesc(sa + 2 * A_TILE + B_TILE);
          wg_fence();
          fence_acc(acc0);
          fence_acc(acc1);
#pragma unroll
          for (int ks = 0; ks < BK / 16; ++ks) {
            const uint64_t off = (uint64_t)((ks * 32) >> 4);
            if constexpr (PASSES == 3) {
              wgmma_n64(acc0, dah + off, dbh + off, 1u);
              wgmma_n64(acc0, dah + off, dbl + off, 1u);
              wgmma_n64(acc0, dal + off, dbh + off, 1u);
              wgmma_n64(acc1, dah + 512 + off, dbh + off, 1u);  // +8192 bytes: rows 64-127
              wgmma_n64(acc1, dah + 512 + off, dbl + off, 1u);
              wgmma_n64(acc1, dal + 512 + off, dbh + off, 1u);
            } else {
              wgmma_n64(acc0, dah + off, dbh + off, 1u);
              wgmma_n64(acc1, dah + 512 + off, dbh + off, 1u);
            }
          }
          wg_commit();
          fence_acc(acc0);
          fence_acc(acc1);
          wg_wait<1>();
          fence_acc(acc0);
          fence_acc(acc1);
          if (prev >= 0) release(prev);
          prev = stage;
          if (++stage == STAGES) { stage = 0; phase_bit ^= 1; }
        }
        wg_wait<0>();
        fence_acc(acc0);
        fence_acc(acc1);
        if (prev >= 0) release(prev);
        // fragments -> [128 x 64] staging (row rr, float4 chunk c at rr * 16 + (c ^ (rr & 15))) -> one row per thread
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
          const int rr = frag_row(ew, lane, j), cc = frag_col(lane, j);
          float* b0 = reinterpret_cast<float*>(accs + rr * 16 + ((cc >> 2) ^ (rr & 15))) + (cc & 3);
          float* b1 = reinterpret_cast<float*>(accs + (rr + 64) * 16 + ((cc >> 2) ^ ((rr + 64) & 15))) + (cc & 3);
          *reinterpret_cast<float2*>(b0) = make_float2(acc0[j], acc0[j + 1]);
          *reinterpret_cast<float2*>(b1) = make_float2(acc1[j], acc1[j + 1]);
        }
        named_sync(1, 128);
#pragma unroll 1
        for (int ch = 0; ch < BN / 32; ++ch) {
          if (ch + 1 < BN / 32) prefetch32(P, r, nt * BN + (ch + 1) * 32, valid, nxt);
          uint32_t v[32];
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            const float4 x = accs[rl * 16 + ((ch * 8 + c) ^ (rl & 15))];
            v[4 * c] = __float_as_uint(x.x); v[4 * c + 1] = __float_as_uint(x.y);
            v[4 * c + 2] = __float_as_uint(x.z); v[4 * c + 3] = __float_as_uint(x.w);
          }
          if (valid) epilogue32(P, r, ti, ug, lr, nt * BN + ch * 32, v, cur);
          cur = nxt;
        }
        named_sync(1, 128);  // staging buffer read by every thread before the next tile overwrites it
      }
    }
    // the producer and the consumers keep separate copies of (stage, phase_bit): both advance them by exactly the same
    // amounts per phase, so no exchange is needed.
    if (P.sync_after) grid_barrier(barrier_ctr, gen, gridDim.x);
    else __syncthreads();  // the next entry is independent of this one: only the descriptor slot is recycled
  }
  __syncthreads();
  if (cs > 1) cluster_sync_all();  // nobody exits while a peer may still multicast into / arrive on its smem
}

// x [rows, 80] fp32 -> planes [rows, 128] (columns 80..127 zero), all rows
__global__ void k_x80_planes(const float* x, int64_t rows, __half* hi, __half* lo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * 128) return;
  const int64_t r = i >> 7;
  const int c = (int)(i & 127);
  const float v = c < 80 ? x[r * 80 + c] : 0.f;
  const __half h = __float2half_rn(v);
  hi[i] = h;
  lo[i] = __float2half_rn(v - __half2float(h));
}

}  // namespace

int x80_planes(Ctx& ctx, const float* x, int64_t rows, __half* hi, __half* lo) {
  if (ctx.dry || rows == 0) return 0;
  k_x80_planes<<<(unsigned)((rows * 128 + 255) / 256), 256, 0, ctx.stream>>>(x, rows, hi, lo);
  SSB_CUDA(cudaGetLastError());
  ++g_launches;
  return 0;
}

int sampler_tc_max_clusters(int cs) {
  // per device: the shared-memory attribute and the occupancy answer belong to the device that is current
  static std::mutex mu;
  static int cache_all[64][9];
  static bool init[64];
  if (cs < 1 || cs > 8) return 0;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  std::lock_guard<std::mutex> lk(mu);
  int* cache = cache_all[dev];
  if (!init[dev]) {
    for (int i = 0; i < 9; ++i) cache[i] = -1;
    init[dev] = true;
  }
  if (cache[cs] >= 0) return cache[cs];
  // both pass counts have the same shared memory and launch bounds: one occupancy answer serves both
  cudaFuncSetAttribute(sampler_tc_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
  cudaFuncSetAttribute(sampler_tc_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(sms / cs * cs));
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = SMEM;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = (unsigned)cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, sampler_tc_kernel<3>, &cfg) != cudaSuccess) { cudaGetLastError(); n = 0; }
  cache[cs] = n;
  return n;
}

int sampler_tc_max_ctas() { return sampler_tc_max_clusters(1); }

int launch_sampler_tc(Ctx& ctx, const CUtensorMap* maps_dev, const SPhase* phases_dev, int nphases, const SeqDev& s,
                      int max_nt, unsigned* barrier_ctr, int cs, bool single_pass) {
  const int ntiles = s.ntiles;
  if (ctx.dry) return 0;
  const int cap = sampler_tc_max_clusters(cs);
  SSB_CHECK(cap > 0, "persistent sampler kernel cannot be resident on this device");
  int ncl = ntiles * (max_nt / cs);
  if (ncl > cap) ncl = cap;
  SSB_CUDA(cudaMemsetAsync(barrier_ctr, 0, sizeof(unsigned), ctx.stream));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(ncl * cs));
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = SMEM;
  cfg.stream = ctx.stream;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = 1;
  at[1].id = cudaLaunchAttributeClusterDimension;
  at[1].val.clusterDim.x = (unsigned)cs; at[1].val.clusterDim.y = 1; at[1].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 2;
  SSB_CUDA(cudaLaunchKernelEx(&cfg, single_pass ? sampler_tc_kernel<1> : sampler_tc_kernel<3>, maps_dev, phases_dev, nphases, s.tiles, s.tile_pos, s.rng, ntiles,
                              barrier_ctr, cs));
  ++g_launches;
  return 0;
}

}  // namespace ssb
