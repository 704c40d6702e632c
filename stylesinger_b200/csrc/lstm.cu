// f3 (SURVEY.md section 8f): the emotion-encoder half of the reference-audio front-end.
//   EmotionEncoder (reference data_gen/tts/emotion/model.py:10-77): a 3-layer batch-first LSTM (40 -> 256 -> 256 -> 256) run
//   from zero state over 160-frame partial utterances; `inference` returns hidden[-1] (model.py:62-77), `forward` adds
//   relu(linear) + L2 normalisation (model.py:51-57); embed_utterance (data_gen/tts/emotion/inference.py:150-151) averages
//   the partial embeddings and L2-normalises.  The result is the `emo_embed` input of the hot path (inference/StyleSinger.py:106).
// As kernels (fp32 FFMA; the recurrence is latency-bound, 480 dependent steps of a 1024 x 256 mat-vec per partial):
//   * per layer the input projection of ALL frames is one plain GEMM  xproj = x W_ih^T + (b_ih + b_hh)   [P T, 1024];
//   * the recurrence runs on one 8-CTA thread-block CLUSTER per group of up to 8 partials: CTA r keeps the W_hh rows of
//     hidden units 32 r .. 32 r + 31 (all four gates, 128 x 256 fp32 = 128 KB) resident in its REGISTER FILE for the whole
//     sequence (128 registers per thread), computes those gates for every partial of the group, applies the cell update and
//     writes its 32 new h values into the (double-buffered) h vector of all 8 CTAs through distributed shared memory
//     (mbarrier-signalled `st.async`, no cluster-wide barrier per frame).  W_hh is read from HBM once per layer instead
//     of once per frame.
#include <cooperative_groups.h>
#include <math.h>
#include <stdlib.h>

#include <memory>
#include <vector>

#include "../../include/stylesinger_b200.h"
#include "common.cuh"
#include "model.cuh"

namespace cg = cooperative_groups;

struct ssb_lstm_encoder {
  ssb::DevicePool pool;
  int n_in = 0, hidden = 0, layers = 0, embed = 0;
  std::vector<float*> wih_t;   // per layer [K_l][4H]: W_ih^T with cluster-permuted gate columns
  std::vector<float*> bias;    // per layer [4H]: b_ih + b_hh, same permutation
  std::vector<float*> whh_p;   // per layer [8][H][128]: CTA r's slice, k-major
  float* lin_wt = nullptr;     // [H][E] = linear.weight^T
  float* lin_b = nullptr;      // [E]
};

namespace ssb {
namespace {

constexpr int H = 256;            // hidden units (model_hidden_size, params_model.py)
constexpr int G4 = 4 * H;         // gate rows
constexpr int NCTA = 8;           // cluster size
constexpr int UPC = H / NCTA;     // hidden units per CTA (32)
constexpr int RPC = 4 * UPC;      // gate rows per CTA (128)
constexpr int PB = 8;             // partials per cluster
constexpr int CELL_THREADS = PB * UPC;  // cell role: 8 partials x 32 units = 256 threads

#define RUN(x)                 \
  do {                         \
    int rc_ = (x);             \
    if (rc_ != 0) return rc_;  \
  } while (0)

// column of the permuted gate axis that holds torch gate row `g` (= q * H + u, q in i|f|g|o): CTA u / 32, local row q * 32 + u % 32
inline int perm_col(int g) {
  const int q = g / H, u = g % H;
  return (u / UPC) * RPC + q * UPC + (u % UPC);
}

// C[M, N] = A[M, K] B[K, N] + bias[N]; 64 x 64 tiles, 4 x 4 per thread, fp32 FFMA.  N % 64 == 0.
__global__ void __launch_bounds__(256) k_gemm_bias(const float* __restrict__ A, const float* __restrict__ B, const float* __restrict__ bias,
                                                   float* __restrict__ Cm, int64_t M, int N, int K) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t m0 = (int64_t)blockIdx.y * 64;
  const int n0 = blockIdx.x * 64;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int r = i >> 4, kk = i & 15;
      const int64_t m = m0 + r;
      As[kk][r] = (m < M && k0 + kk < K) ? A[m * K + k0 + kk] : 0.f;
    }
    for (int i = threadIdx.x; i < 16 * 64; i += 256) {
      const int kk = i >> 6, c = i & 63;
      Bs[kk][c] = (k0 + kk < K) ? B[(int64_t)(k0 + kk) * N + n0 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      Cm[m * N + n] = acc[i][j] + bias[n];
    }
  }
}

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t map_rank(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
// 4-byte store into another CTA's shared memory that reports its bytes to an mbarrier of that CTA
__device__ __forceinline__ void st_async_f32(uint32_t dst_cluster, float v, uint32_t bar_cluster) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(dst_cluster),
               "r"(__float_as_uint(v)), "r"(bar_cluster)
               : "memory");
}
__device__ __forceinline__ void hbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  const long long t0 = clock64();
  while (true) {
    asm volatile(
        "{\n.reg .pred p;\nmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    if (clock64() - t0 > 4000000000LL) __trap();  // ~2 s watchdog: fail loudly instead of hanging the GPU
  }
}

// One LSTM layer over T frames for partials [PB * cluster, ...).  xproj [P, T, 4H] (permuted gate columns, biases folded in),
// whh_p [8][H][128].  hseq [P, T, H] (may be null) receives every h_t, hlast [P, H] (may be null) the final one.
// Mat-vec role: thread (row, kh) keeps W_hh[row][kh * 128 .. + 128) in REGISTERS for the whole sequence (the CTA's 128 KB
// slice = 128 registers per thread) and multiplies it with the h vectors of all 8 partials, read as broadcast float4s from
// shared memory: per frame the SM issues 8 x 128 x 256 FFMAs and only 16 KB of shared-memory reads.
// Cell role: warp `up` = partial, lane `uj` = hidden unit 32 r + uj (c in a register for the whole sequence): sums the two K
// halves and the input projection (fetched one frame ahead), applies the gates, stores h_t into every CTA of the cluster.
// Exchange of h_t: `st.async` stores that report their bytes to an mbarrier of the receiving CTA (one per h buffer, 8 KB
// expected per frame); a CTA starts frame t + 1 as soon as ITS copy of h_t is complete - no cluster-wide barrier.  Double
// buffering is enough: h_{t+1} values can only be sent by a CTA that has received all of h_t, i.e. after every CTA has
// finished the mat-vec of frame t - 1 that read the buffer being overwritten.
// KQ = K splits of the mat-vec: RPC * KQ threads, each with H / KQ weights in registers.
constexpr int KQ = 2;
constexpr int LSTM_THREADS = RPC * KQ;
__global__ void __cluster_dims__(NCTA, 1, 1) __launch_bounds__(LSTM_THREADS, 1)
    k_lstm_layer(const float* __restrict__ xproj, const float* __restrict__ whh_p, int P, int T, float* __restrict__ hseq,
                 float* __restrict__ hlast) {
  __shared__ __align__(16) float hsm[2 * H * PB];   // [2][H][PB]
  constexpr int KH = H / KQ;
  __shared__ float gsm[KQ * PB * RPC];              // [kh][partial][row]
  __shared__ __align__(8) unsigned long long hbar[2];
  cg::cluster_group cl = cg::this_cluster();
  const int r = (int)cl.block_rank();
  const int p0 = (int)(blockIdx.x / NCTA) * PB;
  const int tid = threadIdx.x;
  const int row = tid & (RPC - 1), kh = tid >> 7;
  const int up = tid >> 5, uj = tid & 31;

  float w[KH];
  {
    const float* src = whh_p + ((size_t)r * H + (size_t)kh * KH) * RPC + row;
#pragma unroll
    for (int k = 0; k < KH; ++k) w[k] = src[(size_t)k * RPC];
  }
  for (int i = tid; i < 2 * H * PB; i += LSTM_THREADS) hsm[i] = 0.f;
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(&hbar[0])) : "memory");
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(&hbar[1])) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }

  const bool cell_valid = p0 + up < P;
  const int pc = min(p0 + min(up, PB - 1), P - 1);  // padding partials of the last group recompute the last real one
  const float* xg = xproj + (size_t)pc * T * G4 + (size_t)r * RPC + uj;
  float c_state = 0.f;
  const bool is_cell = tid < CELL_THREADS;
  float nx[4] = {0.f, 0.f, 0.f, 0.f};
  if (is_cell) {
#pragma unroll
    for (int q = 0; q < 4; ++q) nx[q] = xg[q * UPC];
  }
  const uint32_t hsm_a = smem_addr(hsm), bar_a = smem_addr(&hbar[0]);
  cl.sync();  // every CTA of the cluster is resident and has zeroed its h buffers before any remote write

  int cur = 0;
  for (int t = 0; t < T; ++t) {
    float xq[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) xq[q] = nx[q];
    if (is_cell && t + 1 < T) {
#pragma unroll
      for (int q = 0; q < 4; ++q) nx[q] = xg[(size_t)(t + 1) * G4 + q * UPC];
    }
    if (t > 0) hbar_wait(bar_a + 8u * (uint32_t)(t & 1), (uint32_t)(((t - 1) >> 1) & 1));  // h_{t-1} has arrived here
    float acc[PB];
#pragma unroll
    for (int j = 0; j < PB; ++j) acc[j] = 0.f;
    const float4* hc = reinterpret_cast<const float4*>(hsm + (size_t)cur * H * PB + (size_t)kh * KH * PB);
#pragma unroll
    for (int k = 0; k < KH; ++k) {
      const float4 h0 = hc[2 * k], h1 = hc[2 * k + 1];
      acc[0] = fmaf(w[k], h0.x, acc[0]);
      acc[1] = fmaf(w[k], h0.y, acc[1]);
      acc[2] = fmaf(w[k], h0.z, acc[2]);
      acc[3] = fmaf(w[k], h0.w, acc[3]);
      acc[4] = fmaf(w[k], h1.x, acc[4]);
      acc[5] = fmaf(w[k], h1.y, acc[5]);
      acc[6] = fmaf(w[k], h1.z, acc[6]);
      acc[7] = fmaf(w[k], h1.w, acc[7]);
    }
#pragma unroll
    for (int j = 0; j < PB; ++j) gsm[(kh * PB + j) * RPC + row] = acc[j];
    __syncthreads();
    if (tid < CELL_THREADS) {
      const float* g0 = gsm + up * RPC + uj;
      float gs[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float a = g0[q * UPC];
#pragma unroll
        for (int h2 = 1; h2 < KQ; ++h2) a += g0[h2 * PB * RPC + q * UPC];
        gs[q] = xq[q] + a;
      }
      const float gi = gs[0], gf = gs[1], gg = gs[2], go = gs[3];
      c_state = sigmoidf_(gf) * c_state + sigmoidf_(gi) * tanhf(gg);
      const float h = sigmoidf_(go) * tanhf(c_state);
      const int off = (cur ^ 1) * H * PB + (r * UPC + uj) * PB + up;
      if (t + 1 < T) {
        const uint32_t nb = 8u * (uint32_t)((t + 1) & 1);
        // arm the barrier frame t + 1 waits on: everybody's 32 units x 8 partials x 4 bytes.  Its previous phase (frame
        // t - 1) has completed (this thread waited on it); bytes that arrive before the arming are simply counted first
        if (tid == 0)
          asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a + nb), "r"((uint32_t)(H * PB * 4)) : "memory");
#pragma unroll
        for (int d = 0; d < NCTA; ++d)
          st_async_f32(map_rank(hsm_a + 4u * (uint32_t)off, (uint32_t)d), h, map_rank(bar_a + nb, (uint32_t)d));
      }
      if (cell_valid) {
        if (hseq) hseq[((size_t)(p0 + up) * T + t) * H + r * UPC + uj] = h;
        if (hlast && t == T - 1) hlast[(size_t)(p0 + up) * H + r * UPC + uj] = h;
      }
    }
    cur ^= 1;
  }
  cl.sync();  // nobody leaves while a neighbour could still be storing into its shared memory
}

// relu(linear(h)) L2-normalised per partial (model.py:51-57); one block of 256 threads per partial
__global__ void __launch_bounds__(256) k_embed_norm(const float* __restrict__ hid, const float* __restrict__ wt, const float* __restrict__ b,
                                                    int E, float* __restrict__ out) {
  __shared__ float hs[H];
  __shared__ float red[8];
  const int p = blockIdx.x, tid = threadIdx.x;
  hs[tid] = hid[(size_t)p * H + tid];
  __syncthreads();
  float ss = 0.f;
  for (int e = tid; e < E; e += 256) {
    float a = b[e];
    for (int k = 0; k < H; ++k) a = fmaf(hs[k], wt[(size_t)k * E + e], a);
    a = fmaxf(a, 0.f);
    out[(size_t)p * E + e] = a;
    ss += a * a;
  }
  ss = warp_sum(ss);
  if ((tid & 31) == 0) red[tid >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float inv = 1.0f / sqrtf(tot);
  for (int e = tid; e < E; e += 256) out[(size_t)p * E + e] *= inv;
}

// utterance embedding: mean over the utterance's partials, L2-normalised (inference.py:150-151); one block per utterance
__global__ void __launch_bounds__(256) k_utt_embed(const float* __restrict__ hid, const int32_t* __restrict__ offs, float* __restrict__ out) {
  __shared__ float red[8];
  const int u = blockIdx.x, tid = threadIdx.x;
  const int a = offs[u], b = offs[u + 1];
  float s = 0.f;
  for (int p = a; p < b; ++p) s += hid[(size_t)p * H + tid];
  s /= (float)(b - a);
  float ss = warp_sum(s * s);
  if ((tid & 31) == 0) red[tid >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  out[(size_t)u * H + tid] = s / sqrtf(tot);
}

int run_lstm(Ctx& c, const ssb_lstm_encoder& m, const float* frames, int P, int T, const int32_t* utt_offsets_host, int U,
             float* hidden_out, float* embeds_out, float* utt_out) {
  const size_t rows = (size_t)P * T;
  float* xproj = c.alloc<float>(rows * G4);
  float* seq_a = c.alloc<float>(rows * H);
  float* seq_b = c.alloc<float>(rows * H);
  float* hid_ws = c.alloc<float>((size_t)P * H);
  int32_t* offs_dev = c.alloc<int32_t>((size_t)U + 1);
  SSB_CHECK(c.dry || !c.failed, "workspace too small");
  SSB_CHECK((rows + 63) / 64 <= 65535, "too many frames for one call (n_partials * n_frames <= 4 194 240)");
  if (c.dry || P == 0) return 0;
  float* hid = hidden_out ? hidden_out : hid_ws;
  const float* x = frames;
  int K = m.n_in;
  const unsigned groups = (unsigned)((P + PB - 1) / PB);
  for (int l = 0; l < m.layers; ++l) {
    k_gemm_bias<<<dim3(G4 / 64, (unsigned)((rows + 63) / 64)), 256, 0, c.stream>>>(x, m.wih_t[(size_t)l], m.bias[(size_t)l], xproj,
                                                                                   (int64_t)rows, G4, K);
    SSB_CUDA(cudaGetLastError());
    ++g_launches;
    const bool last = l == m.layers - 1;
    float* out_seq = last ? nullptr : ((l & 1) ? seq_b : seq_a);
    float* hl = last ? hid : nullptr;
    const float* wp = m.whh_p[(size_t)l];
    k_lstm_layer<<<groups * NCTA, LSTM_THREADS, 0, c.stream>>>(xproj, wp, P, T, out_seq, hl);
    SSB_CUDA(cudaGetLastError());
    ++g_launches;
    x = out_seq;
    K = H;
  }
  if (embeds_out) {
    k_embed_norm<<<(unsigned)P, 256, 0, c.stream>>>(hid, m.lin_wt, m.lin_b, m.embed, embeds_out);
    SSB_CUDA(cudaGetLastError());
    ++g_launches;
  }
  if (utt_out) {
    SSB_CUDA(cudaMemcpyAsync(offs_dev, utt_offsets_host, sizeof(int32_t) * ((size_t)U + 1), cudaMemcpyHostToDevice, c.stream));
    k_utt_embed<<<(unsigned)U, 256, 0, c.stream>>>(hid, offs_dev, utt_out);
    SSB_CUDA(cudaGetLastError());
    ++g_launches;
  }
  return 0;
}

int check_offsets(const int32_t* offs, int U, int P) {
  SSB_CHECK(offs && U > 0, "utterance offsets missing");
  SSB_CHECK(offs[0] == 0 && offs[U] == P, "utterance offsets must span [0, n_partials]");
  for (int u = 0; u < U; ++u) SSB_CHECK(offs[u + 1] > offs[u], "every utterance needs at least one partial");
  return 0;
}

}  // namespace
}  // namespace ssb

using namespace ssb;

extern "C" {

int ssb_lstm_encoder_create(ssb_lstm_encoder_t** out, int32_t input_size, int32_t hidden_size, int32_t num_layers,
                            const float* const* weight_ih, const float* const* weight_hh, const float* const* bias_ih,
                            const float* const* bias_hh, int32_t embed_size, const float* linear_weight, const float* linear_bias) {
  SSB_CHECK(out, "null argument");
  *out = nullptr;
  SSB_CHECK(weight_ih && weight_hh && bias_ih && bias_hh, "null weight table");
  SSB_CHECK(input_size > 0 && num_layers > 0 && num_layers <= 16, "bad LSTM geometry");
  SSB_CHECK(hidden_size == H, "the cluster LSTM kernel is built for hidden_size 256 (params_model.py: model_hidden_size)");
  SSB_CHECK((linear_weight == nullptr) == (linear_bias == nullptr) && (linear_weight == nullptr || embed_size > 0), "bad linear head");
  std::unique_ptr<ssb_lstm_encoder> m(new ssb_lstm_encoder);
  m->n_in = input_size; m->hidden = hidden_size; m->layers = num_layers; m->embed = linear_weight ? embed_size : 0;
  for (int l = 0; l < num_layers; ++l) {
    SSB_CHECK(weight_ih[l] && weight_hh[l] && bias_ih[l] && bias_hh[l], "null layer weight");
    const int K = l == 0 ? input_size : H;
    std::vector<float> wt((size_t)K * G4), b((size_t)G4), wp((size_t)NCTA * H * RPC);
    for (int g = 0; g < G4; ++g) {
      const int col = perm_col(g);
      for (int k = 0; k < K; ++k) wt[(size_t)k * G4 + col] = weight_ih[l][(size_t)g * K + k];
      b[(size_t)col] = bias_ih[l][g] + bias_hh[l][g];
      const int cta = col / RPC, lr = col % RPC;
      for (int k = 0; k < H; ++k) wp[((size_t)cta * H + k) * RPC + lr] = weight_hh[l][(size_t)g * H + k];
    }
    m->wih_t.push_back(m->pool.upload(wt));
    m->bias.push_back(m->pool.upload(b));
    m->whh_p.push_back(m->pool.upload(wp));
    SSB_CHECK(m->wih_t.back() && m->bias.back() && m->whh_p.back(), "device allocation failed");
  }
  if (linear_weight) {
    std::vector<float> wt((size_t)H * embed_size), b(linear_bias, linear_bias + embed_size);
    for (int e = 0; e < embed_size; ++e)
      for (int k = 0; k < H; ++k) wt[(size_t)k * embed_size + e] = linear_weight[(size_t)e * H + k];
    m->lin_wt = m->pool.upload(wt);
    m->lin_b = m->pool.upload(b);
    SSB_CHECK(m->lin_wt && m->lin_b, "device allocation failed");
  }
  *out = m.release();
  return 0;
}

void ssb_lstm_encoder_free(ssb_lstm_encoder_t* m) { delete m; }

size_t ssb_lstm_encoder_workspace_bytes(const ssb_lstm_encoder_t* m, int32_t n_partials, int32_t n_frames, int32_t n_utterances) {
  if (!m || n_partials < 0 || n_frames <= 0 || n_utterances < 0) return 0;
  Ctx c;
  c.dry = true;
  if (run_lstm(c, *m, nullptr, n_partials, n_frames, nullptr, n_utterances, nullptr, nullptr, nullptr) != 0) return 0;
  return c.high + 4096;
}

int ssb_lstm_encoder_forward(const ssb_lstm_encoder_t* m, const float* frames, int32_t n_partials, int32_t n_frames,
                             const int32_t* utt_offsets, int32_t n_utterances, float* hidden_out, float* embeds_out,
                             float* utt_embed_out, void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && workspace && n_partials >= 0 && n_frames > 0, "bad argument");
  SSB_CHECK(n_partials == 0 || frames, "null frames");
  SSB_CHECK(hidden_out || embeds_out || utt_embed_out, "no output requested");
  SSB_CHECK(!embeds_out || m->lin_wt, "encoder was created without the linear head");
  if (utt_embed_out) RUN(check_offsets(utt_offsets, n_utterances, n_partials));
  Ctx c;
  c.base = (char*)workspace; c.cap = workspace_bytes; c.stream = (cudaStream_t)stream;
  return run_lstm(c, *m, frames, n_partials, n_frames, utt_offsets, utt_embed_out ? n_utterances : 0, hidden_out, embeds_out, utt_embed_out);
}

}  // extern "C"
