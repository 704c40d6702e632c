// Multi-head attention (2 heads x 128) with streaming softmax, fp32.  Rows a3 / a12 of SURVEY.md §8:
//   self-attention of the FFT blocks  (reference modules/commons/common_layers.py:277-286 ->
//   F.multi_head_attention_forward: q*hd^-0.5, bmm, key-padding -> -inf, fp32 softmax, bmm)
//   and the style aligner's cross-attention (reference modules/StyleSinger/lse.py:41).
// The [L,S] score matrix is never materialised (63 MB / utterance / layer in the reference at F=2812).
// One CTA = 64 queries of one (utterance, head); keys/values streamed in tiles of 64.
#include <atomic>

#include "attention.cuh"

namespace ssb {

namespace {

constexpr int BQ = 64, BK = 64, HD = 128;
constexpr int LDT = BQ + 4;  // transposed tiles [d][row]

struct AttnSmem {
  float Qt[HD][LDT];
  float Kt[HD][LDT];
  float Vs[BK][HD];
  float Pt[BK][LDT];
};

__global__ void __launch_bounds__(256, 1) attention_kernel(AttnArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  AttnSmem& sm = *reinterpret_cast<AttnSmem*>(smem_raw);
  const int b = blockIdx.z, head = blockIdx.y;
  const int4 uq = a.utt_q[b], uk = a.utt_k[b];
  const int q0 = blockIdx.x * BQ;
  if (q0 >= uq.y) return;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int nq = min(BQ, uq.y - q0);
  const int hoff = head * HD;

  // load Q tile transposed, scaled
  for (int idx = tid; idx < BQ * HD / 4; idx += 256) {
    const int row = idx & 63, d4 = (idx >> 6) << 2;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row < nq) v = *reinterpret_cast<const float4*>(a.Q + ((int64_t)uq.x + q0 + row) * a.ldq + hoff + d4);
    sm.Qt[d4 + 0][row] = v.x * a.scale;
    sm.Qt[d4 + 1][row] = v.y * a.scale;
    sm.Qt[d4 + 2][row] = v.z * a.scale;
    sm.Qt[d4 + 3][row] = v.w * a.scale;
  }

  float m_run[4], l_run[4], o[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m_run[i] = -INFINITY;
    l_run[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) o[i][j] = 0.f;
  }

  for (int k0 = 0; k0 < uk.y; k0 += BK) {
    const int nkv = min(BK, uk.y - k0);
    __syncthreads();  // previous tile fully consumed (also orders the Q store on the first pass)
    for (int idx = tid; idx < BK * HD / 4; idx += 256) {
      const int row = idx & 63, d4 = (idx >> 6) << 2;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row < nkv) kv = *reinterpret_cast<const float4*>(a.K + ((int64_t)uk.x + k0 + row) * a.ldk + hoff + d4);
      sm.Kt[d4 + 0][row] = kv.x;
      sm.Kt[d4 + 1][row] = kv.y;
      sm.Kt[d4 + 2][row] = kv.z;
      sm.Kt[d4 + 3][row] = kv.w;
    }
    for (int idx = tid; idx < BK * HD / 4; idx += 256) {
      const int row = idx >> 5, d4 = (idx & 31) << 2;
      float4 vv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row < nkv) vv = *reinterpret_cast<const float4*>(a.V + ((int64_t)uk.x + k0 + row) * a.ldv + hoff + d4);
      *reinterpret_cast<float4*>(&sm.Vs[row][d4]) = vv;
    }
    __syncthreads();

    // S = Q K^T : rows ty*4+i, cols tx*4+j
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
    for (int d = 0; d < HD; ++d) {
      const float4 qa = *reinterpret_cast<const float4*>(&sm.Qt[d][ty * 4]);
      const float4 kb = *reinterpret_cast<const float4*>(&sm.Kt[d][tx * 4]);
      const float qv[4] = {qa.x, qa.y, qa.z, qa.w}, kv[4] = {kb.x, kb.y, kb.z, kb.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = fmaf(qv[i], kv[j], s[i][j]);
    }
    // mask
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int kj = tx * 4 + j;
      bool ok = kj < nkv;
      if (ok && a.keymask) ok = a.keymask[(int64_t)uk.x + k0 + kj] != 0.f;
      if (!ok) {
#pragma unroll
        for (int i = 0; i < 4; ++i) s[i][j] = -INFINITY;
      }
    }
    // online softmax (16 lanes of a half-warp share a row group)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mx = fmaxf(fmaxf(s[i][0], s[i][1]), fmaxf(s[i][2], s[i][3]));
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      const float m_new = fmaxf(m_run[i], mx);
      const float m_use = m_new == -INFINITY ? 0.f : m_new;
      float rs = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[i][j] = expf(s[i][j] - m_use);
        rs += s[i][j];
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, off);
      const float corr = m_run[i] == -INFINITY ? 0.f : expf(m_run[i] - m_use);
      l_run[i] = l_run[i] * corr + rs;
      m_run[i] = m_new;
#pragma unroll
      for (int j = 0; j < 8; ++j) o[i][j] *= corr;
    }
    // P^T to smem
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int i = 0; i < 4; ++i) sm.Pt[tx * 4 + j][ty * 4 + i] = s[i][j];
    __syncthreads();
    // O += P V : rows ty*4+i, cols {tx*4+c, 64+tx*4+c}
#pragma unroll 8
    for (int j = 0; j < BK; ++j) {
      const float4 pa = *reinterpret_cast<const float4*>(&sm.Pt[j][ty * 4]);
      const float4 v0 = *reinterpret_cast<const float4*>(&sm.Vs[j][tx * 4]);
      const float4 v1 = *reinterpret_cast<const float4*>(&sm.Vs[j][64 + tx * 4]);
      const float pv[4] = {pa.x, pa.y, pa.z, pa.w};
      const float vv[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int c = 0; c < 8; ++c) o[i][c] = fmaf(pv[i], vv[c], o[i][c]);
    }
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = ty * 4 + i;
    if (row >= nq) continue;
    const float inv = 1.0f / l_run[i];  // no valid key: l = 0 and o = 0, so the row is NaN (attention_tc.cu does the same)
    float* dst = a.out + ((int64_t)uq.x + q0 + row) * a.ldo + hoff;
    *reinterpret_cast<float4*>(dst + tx * 4) = make_float4(o[i][0] * inv, o[i][1] * inv, o[i][2] * inv, o[i][3] * inv);
    *reinterpret_cast<float4*>(dst + 64 + tx * 4) = make_float4(o[i][4] * inv, o[i][5] * inv, o[i][6] * inv, o[i][7] * inv);
  }
}

}  // namespace

std::atomic<long long> g_attn_launches[2];

int attention_check(const AttnArgs& a) {
  SSB_CHECK(a.heads == 1 || a.heads == 2, "attention: heads must be 1 or 2, got " + std::to_string(a.heads));
  SSB_CHECK(a.B >= 0 && a.B <= 65535, "attention: B = " + std::to_string(a.B) + " exceeds gridDim.z (65535)");
  SSB_CHECK(a.out != nullptr, "attention: no output");
  SSB_CHECK(a.ldq % 4 == 0 && a.ldk % 4 == 0 && a.ldv % 4 == 0 && a.ldo % 4 == 0,
            "attention: ldq / ldk / ldv / ldo must be multiples of 4 (float4 loads and stores)");
  SSB_CHECK(((uintptr_t)a.Q | (uintptr_t)a.K | (uintptr_t)a.V | (uintptr_t)a.out) % 16 == 0,
            "attention: Q, K, V and out must be 16-byte aligned (float4 loads and stores)");
  const int w = a.heads * HD;
  SSB_CHECK(a.ldq >= w && a.ldk >= w && a.ldv >= w && a.ldo >= w,
            "attention: an ld is narrower than heads x 128 = " + std::to_string(w) + " columns");
  return 0;
}

int attention(Ctx& ctx, const AttnArgs& a) {
  if (attention_check(a)) return -1;
  if (ctx.dry || a.B == 0 || a.max_q == 0) return 0;
  {  // the attribute is per device (one process may drive several GPUs)
    static std::atomic<bool> configured[64];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!configured[dev].load(std::memory_order_acquire)) {
      SSB_CUDA(cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(AttnSmem)));
      configured[dev].store(true, std::memory_order_release);
    }
  }
  dim3 grid((a.max_q + BQ - 1) / BQ, a.heads, a.B);
  attention_kernel<<<grid, 256, sizeof(AttnSmem), ctx.stream>>>(a);
  SSB_CUDA(cudaGetLastError());
  ++g_launches;
  ++g_attn_launches[0];
  return 0;
}

}  // namespace ssb
