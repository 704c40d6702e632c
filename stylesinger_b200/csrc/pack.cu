// Weight packing: reference state_dict tensors (host, torch layouts) -> device buffers in the layouts the
// kernels consume.  Replaces the reference's module construction + load_ckpt + remove_weight_norm
// (modules/StyleSinger/stylesinger.py:46-117, utils/commons/ckpt_utils.py:26-67,
//  modules/hifigan/hifigan_nsf.py:171-178).
#include <math.h>
#include <string.h>

#include "model.cuh"

namespace ssb {

std::atomic<long long> g_launches{0};
static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
const char* last_error() { return g_err.c_str(); }

DevicePool::~DevicePool() {
  for (void* p : ptrs) cudaFree(p);
}
float* DevicePool::alloc(size_t n) {
  void* p = nullptr;
  if (cudaMalloc(&p, (n ? n : 1) * sizeof(float)) != cudaSuccess) return nullptr;
  ptrs.push_back(p);
  return (float*)p;
}
void DevicePool::release(void* p) {
  if (!p) return;
  for (size_t i = 0; i < ptrs.size(); ++i)
    if (ptrs[i] == p) {
      cudaFree(p);  // synchronises the device: no kernel can still be reading the buffer
      ptrs[i] = ptrs.back();
      ptrs.pop_back();
      return;
    }
}
float* DevicePool::upload(const std::vector<float>& h) {
  float* d = alloc(h.size());
  if (!d) return nullptr;
  if (cudaMemcpy(d, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
  return d;
}

const HostTensor* TensorMap::get(const std::string& name, std::initializer_list<int64_t> shape) {
  auto it = t.find(name);
  if (it == t.end()) {
    if (missing.empty()) missing = "missing tensor '" + name + "'";
    return nullptr;
  }
  if (shape.size()) {
    std::vector<int64_t> s(shape);
    if (s != it->second.shape) {
      if (missing.empty()) missing = "tensor '" + name + "' has an unexpected shape";
      return nullptr;
    }
  }
  return &it->second;
}

static inline int perm_col(int n, int N, PackMode mode) {
  if (mode == PACK_PLAIN) return n;
  const int C = N / 2;
  if (mode == PACK_GATE_SIG_TANH) return n < C ? 2 * n : 2 * (n - C) + 1;  // sigmoid half first
  return n < C ? 2 * n + 1 : 2 * (n - C);                                  // WN: tanh half first
}

// fold torch.nn.utils.weight_norm (dim=0): w = v * (g / ||v||), norm over all dims but 0
static void fold_weight_norm(const HostTensor* v, const HostTensor* g, std::vector<float>& w) {
  const int64_t N = v->shape[0], per = v->numel() / N;
  w.resize(v->numel());
  for (int64_t n = 0; n < N; ++n) {
    double s = 0.0;
    for (int64_t i = 0; i < per; ++i) s += (double)v->data[n * per + i] * v->data[n * per + i];
    const float scale = g->data[n] / (float)sqrt(s);
    for (int64_t i = 0; i < per; ++i) w[n * per + i] = v->data[n * per + i] * scale;
  }
}

// cin16: the layer runs on conv_gemm, which takes Cin % 16 == 0 only (false: a layer only the vocoder's conv_post_tanh reads)
static int pack_from_host(DevicePool& pool, const float* w, int N, int Cin, int k, const float* b, int dil, PackMode mode,
                          Conv* out, bool cin16 = true) {
  SSB_CHECK(!cin16 || Cin % 16 == 0, "pack: Cin must be a multiple of 16");
  const int Npad = (N + 3) & ~3;
  std::vector<float> W((size_t)k * Cin * Npad, 0.f), B((size_t)Npad, 0.f);
  for (int n = 0; n < N; ++n) {
    const int pn = perm_col(n, N, mode);
    for (int c = 0; c < Cin; ++c)
      for (int j = 0; j < k; ++j) W[((size_t)j * Cin + c) * Npad + pn] = w[((size_t)n * Cin + c) * k + j];
    if (b) B[pn] = b[n];
  }
  out->W = pool.upload(W);
  out->bias = b ? pool.upload(B) : nullptr;
  SSB_CHECK(out->W != nullptr && (!b || out->bias != nullptr), "pack: device allocation failed");
  out->taps = k; out->Cin = Cin; out->N = N; out->Npad = Npad; out->dil = dil; out->center = (k - 1) / 2;
  return 0;
}

static int pack_conv_impl(DevicePool& pool, const HostTensor* w, const HostTensor* b, int dil, PackMode mode, Conv* out,
                          const HostTensor* g, bool cin16) {
  if (!w) return -1;
  SSB_CHECK(w->shape.size() == 3 || w->shape.size() == 2, "pack_conv: weight must be [N,Cin,k] or [N,Cin]");
  const int N = (int)w->shape[0], Cin = (int)w->shape[1], k = w->shape.size() == 3 ? (int)w->shape[2] : 1;
  std::vector<float> folded;
  const float* src = w->data;
  if (g) {
    fold_weight_norm(w, g, folded);
    src = folded.data();
  }
  return pack_from_host(pool, src, N, Cin, k, b ? b->data : nullptr, dil, mode, out, cin16);
}

int pack_conv(DevicePool& pool, const HostTensor* w, const HostTensor* b, int dil, PackMode mode, Conv* out,
              const HostTensor* g) {
  return pack_conv_impl(pool, w, b, dil, mode, out, g, true);
}

// Power-of-two exponent s for the planes of W * 2^s: s = 14 - ceil(log2 max|w|), so that max|W * 2^s| <= 2^14 and the lo
// plane of every weight above max|w| * 2^-16 is a normal fp16 number (conv_gemm_tc.cuh, "Precision").  0 for an all-zero
// (or non-finite) tensor; clamped so that 2^-s stays a normal fp32 number.
static int plane_exponent(const float* w, size_t n) {
  float mx = 0.f;
  for (size_t i = 0; i < n; ++i) mx = fmaxf(mx, fabsf(w[i]));
  if (!(mx > 0.f) || mx == HUGE_VALF) return 0;  // (fmaxf drops NaNs)
  int e = 0;
  const float m = frexpf(mx, &e);  // mx = m * 2^e, m in [0.5, 1): ceil(log2 mx) = e, or e - 1 when mx is a power of two
  const int s = 14 - (m == 0.5f ? e - 1 : e);
  return s < -126 ? -126 : (s > 126 ? 126 : s);
}

// Tensor-core packing: W[tap][n'][c] * 2^s as fp16 hi/lo planes (n' = permuted output column), wscale = 2^-s, + TMA maps.
int pack_conv_tc(DevicePool& pool, const HostTensor* w, int dil, PackMode mode, const float* packed_bias, ConvTC* out) {
  if (!w) return -1;
  const int N = (int)w->shape[0], Cin = (int)w->shape[1], k = w->shape.size() == 3 ? (int)w->shape[2] : 1;
  if (Cin % 64 != 0 || N % 64 != 0 || !tc_available()) return 0;  // not eligible: out->ok stays false
  const int s = plane_exponent(w->data, (size_t)k * N * Cin);
  std::vector<__half> hi((size_t)k * N * Cin), lo((size_t)k * N * Cin);
  for (int n = 0; n < N; ++n) {
    const int pn = perm_col(n, N, mode);
    for (int c = 0; c < Cin; ++c)
      for (int j = 0; j < k; ++j) {
        const float v = ldexpf(w->data[((size_t)n * Cin + c) * k + j], s);  // exact: a power-of-two scale
        const __half h = __float2half_rn(v);
        const size_t o = ((size_t)j * N + pn) * Cin + c;
        hi[o] = h;
        lo[o] = __float2half_rn(v - __half2float(h));
      }
  }
  void *dh = nullptr, *dl = nullptr;
  SSB_CUDA(cudaMalloc(&dh, hi.size() * sizeof(__half)));
  pool.ptrs.push_back(dh);
  SSB_CUDA(cudaMalloc(&dl, lo.size() * sizeof(__half)));
  pool.ptrs.push_back(dl);
  SSB_CUDA(cudaMemcpy(dh, hi.data(), hi.size() * sizeof(__half), cudaMemcpyHostToDevice));
  SSB_CUDA(cudaMemcpy(dl, lo.data(), lo.size() * sizeof(__half), cudaMemcpyHostToDevice));
  out->W_hi = (__half*)dh; out->W_lo = (__half*)dl;
  out->taps = k; out->Cin = Cin; out->N = N; out->dil = dil; out->center = (k - 1) / 2; out->bias = packed_bias;
  out->wscale = ldexpf(1.0f, -s);
  return make_weight_maps(out);
}

int pack_dense(DevicePool& pool, const HostTensor* w, const HostTensor* b, int dil, PackMode mode, Dense* out,
               const HostTensor* g, int row0, int nrows) {
  if (!w) return -1;
  SSB_CHECK(w->shape.size() == 3 || w->shape.size() == 2, "pack_dense: weight must be [N,Cin,k] or [N,Cin]");
  const int Cin = (int)w->shape[1], k = w->shape.size() == 3 ? (int)w->shape[2] : 1;
  if (nrows < 0) nrows = (int)w->shape[0] - row0;
  std::vector<float> folded;
  const float* src = w->data;
  if (g) {
    fold_weight_norm(w, g, folded);
    src = folded.data();
  }
  src += (size_t)row0 * Cin * k;
  if (pack_from_host(pool, src, nrows, Cin, k, b ? b->data + row0 : nullptr, dil, mode, &out->f)) return -1;
  HostTensor t;  // the tensor-core packer reads the torch conv layout [N, Cin, k]; its bias is the packed fp32 vector
  t.data = src;
  t.shape = {nrows, Cin, k};
  return pack_conv_tc(pool, &t, dil, mode, out->f.bias, &out->t);
}
// Narrow convs (C = 64 / G channels, G = 2, 4, 8) on the 64-wide K block: view [rows, C] as [rows/G, 64] (G consecutive
// time steps per "super row", super channel = phase*C + c).  y[Gq+phi, n] = sum_j sum_c W[n][c][j] x[Gq + phi + s_j, c]
// with s_j = (j - cen)*d becomes a conv over super rows:
//  * G does not divide d: taps delta = floor((phi + s_j)/G) with input phase (phi + s_j) mod G, the dense tap range
//    [-ceil(cen*d/G), ceil(cen*d/G)] at dilation 1:  W'[delta][phi'*C + c][phi*C + n] = W[n][c][j];
//  * G divides d: s_j moves every phase by the same (j - cen)*d/G super rows, so the conv keeps its k taps at dilation
//    d/G and is block-diagonal over the phases:  W'[j][phi*C + c][phi*C + n] = W[n][c][j]  (7 taps instead of up to 37
//    for HiFi-GAN V3's dilation 12 at C = 32).
// Most of each 64x64 block is zero, which the tensor cores absorb easily (the fp32 FFMA kernel ran the C = 32 convs at
// ~15 TFLOP/s ungrouped).  The tensor-core packing goes to out->t; with ffma also the FFMA one to out->f (C = 16, 8:
// conv_gemm takes Cin % 16 == 0, and one grouped path serves both GEMMs).  At G = 2 a shape the packing does not take
// (an even kernel) leaves out->t.ok false and the stage runs ungrouped on FFMA; at G > 2 it is an error.
static int pack_conv_grouped(DevicePool& pool, const HostTensor* v, const HostTensor* g, int dil, int G, const float* bias_host,
                             bool ffma, Dense* out) {
  if (!v || !g) return -1;
  const int C = 64 / G;
  const int N = (int)v->shape[0], Cin = (int)v->shape[1], k = v->shape.size() == 3 ? (int)v->shape[2] : 0;
  const bool ok = v->shape.size() == 3 && N == C && Cin == C && k % 2 == 1;
  if (!ok && G == 2) return 0;
  SSB_CHECK(ok, "ssb_vocoder_create: a ResBlock conv of a " + std::to_string(C) + "-channel stage must be [" +
                    std::to_string(C) + ", " + std::to_string(C) + ", k] with k odd");
  std::vector<float> w;
  fold_weight_norm(v, g, w);
  const int cen = (k - 1) / 2;
  const bool dilated = dil % G == 0;
  auto fdiv = [G](int a) { return a >= 0 ? a / G : -((-a + G - 1) / G); };  // floor(a / G)
  const int dmin = dilated ? -cen : fdiv(-cen * dil), dmax = dilated ? cen : fdiv(G - 1 + cen * dil);
  const int taps = dmax - dmin + 1;
  std::vector<float> t((size_t)64 * 64 * taps, 0.f);  // torch conv layout [N'=64][Cin'=64][taps]
  for (int phi = 0; phi < G; ++phi)
    for (int j = 0; j < k; ++j) {
      const int s = (j - cen) * dil;
      const int delta = dilated ? j - cen : fdiv(phi + s), ph_in = dilated ? phi : (phi + s) - G * delta;
      for (int n = 0; n < C; ++n)
        for (int c = 0; c < C; ++c)
          t[((size_t)(phi * C + n) * 64 + (ph_in * C + c)) * taps + (delta - dmin)] = w[((size_t)n * C + c) * k + j];
    }
  const int dil_g = dilated ? dil / G : 1;
  std::vector<float> b2(64, 0.f);
  if (bias_host)
    for (int i = 0; i < 64; ++i) b2[i] = bias_host[i % C];
  const float* bias_dev = nullptr;
  if (ffma) {
    if (pack_from_host(pool, t.data(), 64, 64, taps, b2.data(), dil_g, PACK_PLAIN, &out->f)) return -1;
    bias_dev = out->f.bias;
  } else {
    bias_dev = pool.upload(b2);
  }
  HostTensor ht;
  ht.data = t.data();
  ht.shape = {64, 64, taps};
  if (pack_conv_tc(pool, &ht, dil_g, PACK_PLAIN, bias_dev, &out->t)) return -1;
  if (out->t.ok && out->t.center != -dmin) return -1;  // symmetric by construction
  return 0;
}

// weight-normed ConvTranspose1d (k = 2u) -> 3-tap conv with N = u*Cout -> tensor-core packing
static int pack_conv_transpose_tc(DevicePool& pool, const HostTensor* v, const HostTensor* g, int u, const float* packed_bias, ConvTC* out) {
  if (!v || !g) return -1;
  const int Cin = (int)v->shape[0], Cout = (int)v->shape[1], k = (int)v->shape[2];
  const int p = (k - u) / 2, N = u * Cout;
  std::vector<float> w;
  fold_weight_norm(v, g, w);
  std::vector<float> t((size_t)N * Cin * 3, 0.f);  // torch conv layout [N][Cin][3]
  for (int phi = 0; phi < u; ++phi)
    for (int j = 0; j < k; ++j) {
      const int num = phi + p - j;
      if (num % u != 0) continue;
      const int d = num / u;
      if (d < -1 || d > 1) return 0;
      for (int c = 0; c < Cin; ++c)
        for (int n = 0; n < Cout; ++n) t[((size_t)(phi * Cout + n) * Cin + c) * 3 + (d + 1)] = w[((size_t)c * Cout + n) * k + j];
    }
  HostTensor ht;
  ht.data = t.data();
  ht.shape = {N, Cin, 3};
  return pack_conv_tc(pool, &ht, 1, PACK_PLAIN, packed_bias, out);
}

int pack_linear(DevicePool& pool, const HostTensor* w, const HostTensor* b, Conv* out) {
  if (!w) return -1;
  return pack_from_host(pool, w->data, (int)w->shape[0], (int)w->shape[1], 1, b ? b->data : nullptr, 1, PACK_PLAIN, out);
}

// ConvTranspose1d(Cin, Cout, k, stride u, padding (k-u)/2) as a 3-tap conv with N = u*Cout:
//   y[q*u + phi, n] = sum_d sum_c x[q + d, c] * w[c, n, phi + p - d*u]      (d in {-1,0,1})
int pack_conv_transpose(DevicePool& pool, const HostTensor* v, const HostTensor* g, const HostTensor* b, int u, Conv* out) {
  if (!v) return -1;
  const int Cin = (int)v->shape[0], Cout = (int)v->shape[1], k = (int)v->shape[2];
  const int p = (k - u) / 2;
  SSB_CHECK(Cin % 16 == 0, "pack_conv_transpose: Cin must be a multiple of 16");
  std::vector<float> w;
  if (g) fold_weight_norm(v, g, w);  // weight_norm dim=0 -> per input channel for ConvTranspose1d
  else w.assign(v->data, v->data + v->numel());
  const int N = u * Cout, Npad = (N + 3) & ~3;
  std::vector<float> W((size_t)3 * Cin * Npad, 0.f), B((size_t)Npad, 0.f);
  for (int phi = 0; phi < u; ++phi)
    for (int j = 0; j < k; ++j) {
      // j = phi + p - d*u  ->  d = (phi + p - j) / u must be an integer in [-1, 1]
      const int num = phi + p - j;
      if (num % u != 0) continue;
      const int d = num / u;
      SSB_CHECK(d >= -1 && d <= 1, "pack_conv_transpose: kernel reach exceeds 3 taps");
      for (int c = 0; c < Cin; ++c)
        for (int n = 0; n < Cout; ++n)
          W[((size_t)(d + 1) * Cin + c) * Npad + phi * Cout + n] = w[((size_t)c * Cout + n) * k + j];
    }
  if (b)
    for (int phi = 0; phi < u; ++phi)
      for (int n = 0; n < Cout; ++n) B[phi * Cout + n] = b->data[n];
  out->W = pool.upload(W);
  out->bias = pool.upload(B);
  SSB_CHECK(out->W && out->bias, "pack_conv_transpose: device allocation failed");
  out->taps = 3; out->Cin = Cin; out->N = N; out->Npad = Npad; out->dil = 1; out->center = 1;
  return 0;
}

static float* upload_tensor(DevicePool& pool, const HostTensor* t) {
  if (!t) return nullptr;
  std::vector<float> h(t->data, t->data + t->numel());
  return pool.upload(h);
}

#define PK(expr)                 \
  do {                           \
    if ((expr) != 0) goto fail;  \
  } while (0)

static int build_fft(TensorMap& tm, DevicePool& pool, const std::string& p, int n_layers, int k, bool pos_alpha, FFT* f) {
  f->kernel = k;
  f->layers.resize(n_layers);
  for (int i = 0; i < n_layers; ++i) {
    const std::string q = p + "layers." + std::to_string(i) + ".op.";
    FFTLayer& L = f->layers[i];
    L.ln1_g = upload_tensor(pool, tm.get(q + "layer_norm1.weight"));
    L.ln1_b = upload_tensor(pool, tm.get(q + "layer_norm1.bias"));
    L.ln2_g = upload_tensor(pool, tm.get(q + "layer_norm2.weight"));
    L.ln2_b = upload_tensor(pool, tm.get(q + "layer_norm2.bias"));
    // in_proj [3H, H] / out_proj [H, H], bias-free (common_layers.py:200-205)
    if (pack_dense(pool, tm.get(q + "self_attn.in_proj_weight"), nullptr, 1, PACK_PLAIN, &L.qkv)) return -1;
    if (pack_dense(pool, tm.get(q + "self_attn.out_proj.weight"), nullptr, 1, PACK_PLAIN, &L.out)) return -1;
    if (pack_dense(pool, tm.get(q + "ffn.ffn_1.weight"), tm.get(q + "ffn.ffn_1.bias"), 1, PACK_PLAIN, &L.ffn1)) return -1;
    if (pack_dense(pool, tm.get(q + "ffn.ffn_2.weight"), tm.get(q + "ffn.ffn_2.bias"), 1, PACK_PLAIN, &L.ffn2)) return -1;
    f->tc_ok = f->tc_ok && L.qkv.t.ok && L.out.t.ok && L.ffn1.t.ok && L.ffn2.t.ok;
  }
  f->ln_g = upload_tensor(pool, tm.get(p + "layer_norm.weight"));
  f->ln_b = upload_tensor(pool, tm.get(p + "layer_norm.bias"));
  f->pos_alpha = pos_alpha ? upload_tensor(pool, tm.get(p + "pos_embed_alpha")) : nullptr;
  return 0;
}

static int build_denoiser(TensorMap& tm, DevicePool& pool, const std::string& p, int C, int L, int cycle, int in_dims,
                          int out_dims, bool ddiff, Denoiser* d) {
  d->C = C; d->L = L; d->cycle = cycle; d->in_dims = in_dims; d->out_dims = out_dims; d->ddiff = ddiff;
  if (ddiff) {
    d->in_w = upload_tensor(pool, tm.get(p + "input_projection.weight"));
    d->in_b = upload_tensor(pool, tm.get(p + "input_projection.bias"));
    d->uv_emb = upload_tensor(pool, tm.get(p + "uv_embed.weight"));
  } else {
    if (pack_conv(pool, tm.get(p + "input_projection.weight"), tm.get(p + "input_projection.bias"), 1, PACK_PLAIN, &d->in_proj)) return -1;
  }
  if (pack_linear(pool, tm.get(p + "mlp.0.weight"), tm.get(p + "mlp.0.bias"), &d->mlp0)) return -1;
  if (pack_linear(pool, tm.get(p + "mlp.2.weight"), tm.get(p + "mlp.2.bias"), &d->mlp2)) return -1;
  d->layers.resize(L);
  const int H = 256;
  const int N2 = 2 * C;
  std::vector<float> Wc((size_t)H * L * N2, 0.f), Bc((size_t)L * N2, 0.f);
  for (int i = 0; i < L; ++i) {
    const std::string q = p + "residual_layers." + std::to_string(i) + ".";
    const int dil = 1 << (i % cycle);
    if (pack_dense(pool, tm.get(q + "dilated_conv.weight"), tm.get(q + "dilated_conv.bias"), dil, PACK_GATE_SIG_TANH, &d->layers[i].dil)) return -1;
    if (pack_dense(pool, tm.get(q + "output_projection.weight"), tm.get(q + "output_projection.bias"), 1, PACK_PLAIN, &d->layers[i].outp)) return -1;
    if (pack_linear(pool, tm.get(q + "diffusion_projection.weight"), tm.get(q + "diffusion_projection.bias"), &d->layers[i].dproj)) return -1;
    const HostTensor* cw = tm.get(q + "conditioner_projection.weight");
    const HostTensor* cb = tm.get(q + "conditioner_projection.bias");
    if (!cw || !cb) return -1;
    for (int n = 0; n < N2; ++n) {
      const int pn = i * N2 + perm_col(n, N2, PACK_GATE_SIG_TANH);
      for (int c = 0; c < H; ++c) Wc[(size_t)c * L * N2 + pn] = cw->data[(size_t)n * H + c];
      Bc[pn] = cb->data[n];
    }
    {  // tensor-core path: the gate GEMM's bias (the hoisted conditioner projection below carries none)
      const HostTensor* db = tm.get(q + "dilated_conv.bias");
      if (!db) return -1;
      std::vector<float> bs((size_t)N2);
      for (int n = 0; n < N2; ++n) bs[perm_col(n, N2, PACK_GATE_SIG_TANH)] = db->data[n] + cb->data[n];
      d->layers[i].bias_gate_tc = pool.upload(bs);
    }
  }
  {  // tensor-core packing of the SAME stacked projection (no bias: bias_gate_tc already carries dil + conditioner bias):
     // hoisted out of the T loop, its [rows, L*2C] output is the per-layer addend of the GATE epilogue (EpiTC::add)
    std::vector<float> wt((size_t)L * N2 * H);  // torch layout [N = L*2C][Cin = 256][1], rows in packed column order
    for (int pn = 0; pn < L * N2; ++pn)
      for (int c = 0; c < H; ++c) wt[(size_t)pn * H + c] = Wc[(size_t)c * L * N2 + pn];
    HostTensor ht;
    ht.data = wt.data();
    ht.shape = {L * N2, H, 1};
    if (pack_conv_tc(pool, &ht, 1, PACK_PLAIN, nullptr, &d->cond_all_tc)) return -1;
  }
  d->tc_ok = d->cond_all_tc.ok;
  for (auto& l : d->layers) d->tc_ok = d->tc_ok && l.dil.t.ok && l.outp.t.ok;
  d->cond_all.W = pool.upload(Wc);
  d->cond_all.bias = pool.upload(Bc);
  d->cond_all.taps = 1; d->cond_all.Cin = H; d->cond_all.N = L * N2; d->cond_all.Npad = L * N2; d->cond_all.dil = 1; d->cond_all.center = 0;
  if (pack_conv(pool, tm.get(p + "skip_projection.weight"), tm.get(p + "skip_projection.bias"), 1, PACK_PLAIN, &d->skip_proj)) return -1;
  if (pack_conv(pool, tm.get(p + "output_projection.weight"), tm.get(p + "output_projection.bias"), 1, PACK_PLAIN, &d->out_proj)) return -1;
  if (C % 64 == 0 && in_dims <= 128 && out_dims <= 128) {
    // tensor-core packing of the step's head/tail GEMMs for the persistent sampler.
    // mel net: in_proj K 80->128, skip_proj, out_proj N 80->256.  F0 nets: skip_proj N 192->256, out_proj N 3->128.
    const HostTensor* sw = tm.get(p + "skip_projection.weight");
    const HostTensor* sbias = tm.get(p + "skip_projection.bias");
    const HostTensor* ow = tm.get(p + "output_projection.weight");
    const HostTensor* ob = tm.get(p + "output_projection.bias");
    if (!sw || !sbias || !ow || !ob) return -1;
    const int Ns = (C + 127) / 128 * 128 < 256 ? 256 : (C + 127) / 128 * 128;  // 256 for C = 192 and 256
    const int No = ddiff ? 128 : 256;
    std::vector<float> ws((size_t)Ns * C, 0.f), bs((size_t)Ns, 0.f), wo((size_t)No * C, 0.f), bo((size_t)No, 0.f);
    const float sc = 1.0f / sqrtf((float)L);
    for (int n = 0; n < C; ++n) {
      for (int c = 0; c < C; ++c) ws[(size_t)n * C + c] = sw->data[(size_t)n * C + c] * sc;
      bs[n] = sbias->data[n];
    }
    for (int n = 0; n < out_dims; ++n) {
      for (int c = 0; c < C; ++c) wo[(size_t)n * C + c] = ow->data[(size_t)n * C + c];
      bo[n] = ob->data[n];
    }
    d->out_bias_pad = pool.upload(bo);
    d->skip_bias_pad = pool.upload(bs);
    HostTensor ts, to;
    ts.data = ws.data(); ts.shape = {Ns, C, 1};
    to.data = wo.data(); to.shape = {No, C, 1};
    if (pack_conv_tc(pool, &ts, 1, PACK_PLAIN, d->skip_bias_pad, &d->skip_tc)) return -1;
    if (pack_conv_tc(pool, &to, 1, PACK_PLAIN, d->out_bias_pad, &d->out_tc)) return -1;
    if (!ddiff) {
      const HostTensor* iw = tm.get(p + "input_projection.weight");
      if (!iw) return -1;
      std::vector<float> wi((size_t)C * 128, 0.f);
      for (int n = 0; n < C; ++n)
        for (int c = 0; c < in_dims; ++c) wi[(size_t)n * 128 + c] = iw->data[(size_t)n * in_dims + c];
      HostTensor ti;
      ti.data = wi.data(); ti.shape = {C, 128, 1};
      if (pack_conv_tc(pool, &ti, 1, PACK_PLAIN, d->in_proj.bias, &d->in_tc)) return -1;
    }
  }
  return 0;
}

// PitchPredictor(idim = n_chans = H, n_layers 5, odim 2, kernel_size = predictor_kernel) (stylesinger.py:73-82,
// tts_modules.py:191-219): the convs in both the fp32 and the tensor-core layout, like the decoder's FFN convs
static int build_pitch_predictor(TensorMap& tm, DevicePool& pool, const std::string& p, int H, PitchPredictor* pp) {
  for (int i = 0; i < PitchPredictor::kLayers; ++i) {
    const std::string q = p + "conv." + std::to_string(i) + ".";
    const HostTensor* w = tm.get(q + "1.weight");
    if (!w) return -1;
    const int k = w->shape.size() == 3 ? (int)w->shape[2] : 0;
    SSB_CHECK(w->shape.size() == 3 && w->shape[0] == H && w->shape[1] == H,
              "ssb_model_create: " + q + "1.weight must be [" + std::to_string(H) + ", " + std::to_string(H) + ", k]");
    SSB_CHECK(k % 2 == 1 && (k - 1) / 2 <= GUARD,
              "ssb_model_create: " + q + "1.weight: kernel size " + std::to_string(k) + " must be odd with (k - 1) / 2 <= " +
                  std::to_string(GUARD));
    if (pack_dense(pool, w, tm.get(q + "1.bias", {H}), 1, PACK_PLAIN, &pp->conv[i])) return -1;
    pp->tc_ok = pp->tc_ok && pp->conv[i].t.ok;
    pp->ln_g[i] = upload_tensor(pool, tm.get(q + "3.weight", {H}));
    pp->ln_b[i] = upload_tensor(pool, tm.get(q + "3.bias", {H}));
  }
  if (pack_linear(pool, tm.get(p + "linear.weight", {2, H}), tm.get(p + "linear.bias", {2}), &pp->linear)) return -1;
  pp->pos_alpha = upload_tensor(pool, tm.get(p + "pos_embed_alpha", {1}));
  return 0;
}

int build_model(TensorMap& tm, const ssb_hparams& hp, Model* m, int mel_decoder, int f0_gen, const ssb_model_switches& sw,
                bool use_spk_id) {
  DevicePool& pool = m->pool;
  m->hp = hp;
  m->mel_decoder = mel_decoder;
  m->f0_gen = f0_gen;
  m->sw = sw;
  m->cond_width = cond_width(sw);
  m->spk_id = use_spk_id;
  const bool prodiff = mel_decoder == SSB_MEL_DECODER_PRODIFF;
  const bool fft = mel_decoder == SSB_MEL_DECODER_FFT;
  const int H = hp.hidden_size;
  SSB_CHECK(H == 256, "hidden_size must be 256");
  SSB_CHECK(hp.dur_layers <= 4 && hp.rq_depth <= 8, "unsupported dur_layers / rq_depth");
  {
    const HostTensor* pt = tm.get("__pos_table");
    if (pt) {
      m->pos_table = upload_tensor(pool, pt);
      m->pos_rows = (int)pt->shape[0];
    }
    const HostTensor* te = tm.get("encoder.embed_tokens.weight");
    if (te) {
      m->tok_emb = upload_tensor(pool, te);
      m->n_tokens = (int)te->shape[0];
    }
  }
  m->note_emb = upload_tensor(pool, tm.get("note_encoder.emb.weight", {100, H}));
  m->type_emb = upload_tensor(pool, tm.get("note_encoder.type_emb.weight", {5, H}));
  m->dur_w = upload_tensor(pool, tm.get("note_encoder.dur_ln.weight", {H, 1}));
  m->dur_b = upload_tensor(pool, tm.get("note_encoder.dur_ln.bias", {H}));
  m->pitch_emb = upload_tensor(pool, tm.get("pitch_embed.weight", {300, H}));
  // ProDiffusion.norm_spec / denorm_spec are the identity (prodiff.py:225-229): its spec_min/max go unread; an FFT model
  // has no diffusion at all
  if (!prodiff && !fft) {
    m->spec_min = upload_tensor(pool, tm.get("postdiff.spec_min"));
    m->spec_max = upload_tensor(pool, tm.get("postdiff.spec_max"));
  }
  if (use_spk_id) {
    // Embedding(num_spk + 1, H) (fs2.py:37-38, common_layers.py:62-67): a lookup table, no bias
    const HostTensor* t = tm.get("spk_embed_proj.weight");
    if (!t) goto fail;
    SSB_CHECK(t->shape.size() == 2 && t->shape[0] >= 1 && t->shape[1] == H,
              "ssb_model_create_ex4: with use_spk_id, spk_embed_proj.weight must be [rows, " + std::to_string(H) + "]");
    m->spk_tab = upload_tensor(pool, t);
    m->spk_rows = (int)t->shape[0];
  } else {
    PK(pack_linear(pool, tm.get("spk_embed_proj.weight"), tm.get("spk_embed_proj.bias"), &m->spk_proj));
  }
  if (sw.emo) PK(pack_linear(pool, tm.get("emo_embed_proj.weight"), tm.get("emo_embed_proj.bias"), &m->emo_proj));
  PK(build_fft(tm, pool, "encoder.", hp.enc_layers, hp.enc_ffn_kernel, false, &m->enc));
  PK(build_fft(tm, pool, "decoder.", hp.dec_layers, hp.dec_ffn_kernel, true, &m->dec));
  m->dp_layers = hp.dur_layers;
  for (int i = 0; i < hp.dur_layers; ++i) {
    const std::string q = "dur_predictor.conv." + std::to_string(i) + ".";
    PK(pack_conv(pool, tm.get(q + "1.weight"), tm.get(q + "1.bias"), 1, PACK_PLAIN, &m->dp_conv[i]));
    m->dp_ln_g[i] = upload_tensor(pool, tm.get(q + "3.weight"));
    m->dp_ln_b[i] = upload_tensor(pool, tm.get(q + "3.bias"));
  }
  PK(pack_linear(pool, tm.get("dur_predictor.linear.weight"), tm.get("dur_predictor.linear.bias"), &m->dp_lin));
  // style adaptor, RVQ, l1 and aligner (stylesinger.py:61-64): built only with style
  if (sw.style) {
    for (int i = 0; i < 4; ++i) {
      const std::string a = "style_extractor.wavenet.in_layers." + std::to_string(i) + ".";
      const std::string r = "style_extractor.wavenet.res_skip_layers." + std::to_string(i) + ".";
      PK(pack_conv(pool, tm.get(a + "weight_v"), tm.get(a + "bias"), 1, PACK_GATE_TANH_SIG, &m->wn_in[i], tm.get(a + "weight_g")));
      PK(pack_conv(pool, tm.get(r + "weight_v"), tm.get(r + "bias"), 1, PACK_PLAIN, &m->wn_rs[i], tm.get(r + "weight_g")));
    }
    for (int i = 0; i < 5; ++i)
      for (int j = 0; j < 2; ++j) {
        const std::string q = "style_extractor.encoder.res_blocks." + std::to_string(i) + ".blocks." + std::to_string(j) + ".";
        Model::CB& c = m->cb[i * 2 + j];
        c.ln_g = upload_tensor(pool, tm.get(q + "0.weight"));
        c.ln_b = upload_tensor(pool, tm.get(q + "0.bias"));
        PK(pack_conv(pool, tm.get(q + "1.weight"), tm.get(q + "1.bias"), 1, PACK_PLAIN, &c.c1));
        PK(pack_conv(pool, tm.get(q + "4.weight"), tm.get(q + "4.bias"), 1, PACK_PLAIN, &c.c2));
      }
    m->cb_last_g = upload_tensor(pool, tm.get("style_extractor.encoder.last_norm.weight"));
    m->cb_last_b = upload_tensor(pool, tm.get("style_extractor.encoder.last_norm.bias"));
    PK(pack_conv(pool, tm.get("style_extractor.encoder.post_net1.weight"), tm.get("style_extractor.encoder.post_net1.bias"), 1, PACK_PLAIN, &m->cb_post));
    {
      std::vector<float> cbs((size_t)hp.rq_depth * hp.n_rq * H);
      for (int d = 0; d < hp.rq_depth; ++d) {
        const HostTensor* c = tm.get("style_extractor.rqvae.codebooks." + std::to_string(d) + ".weight", {hp.n_rq + 1, H});
        if (!c) goto fail;
        memcpy(&cbs[(size_t)d * hp.n_rq * H], c->data, sizeof(float) * hp.n_rq * H);  // row n_rq = padding, unused (RQ.py:31)
      }
      m->codebooks = pool.upload(cbs);
      m->cb_norm2 = pool.alloc((size_t)hp.rq_depth * hp.n_rq);
      Ctx c;
      PK(codebook_norms(c, m->codebooks, hp.rq_depth * hp.n_rq, m->cb_norm2));
    }
    PK(pack_linear(pool, tm.get("l1.weight"), tm.get("l1.bias"), &m->l1));
    for (int i = 0; i < 2; ++i) {
      const std::string q = "align.layers." + std::to_string(i) + ".";
      AlignLayer& a = m->align[i];
      const HostTensor* iw = tm.get(q + "multihead_attn.in_proj_weight", {3 * H, H});
      const HostTensor* ib = tm.get(q + "multihead_attn.in_proj_bias", {3 * H});
      PK(pack_dense(pool, iw, ib, 1, PACK_PLAIN, &a.q, nullptr, 0, H));
      PK(pack_dense(pool, iw, ib, 1, PACK_PLAIN, &a.kv, nullptr, H, 2 * H));
      PK(pack_dense(pool, tm.get(q + "multihead_attn.out_proj.weight"), tm.get(q + "multihead_attn.out_proj.bias"), 1, PACK_PLAIN, &a.out));
      PK(pack_dense(pool, tm.get(q + "linear1.weight"), tm.get(q + "linear1.bias"), 1, PACK_PLAIN, &a.lin1));
      PK(pack_dense(pool, tm.get(q + "linear2.weight"), tm.get(q + "linear2.bias"), 1, PACK_PLAIN, &a.lin2));
      m->align_tc_ok = m->align_tc_ok && a.q.t.ok && a.kv.t.ok && a.out.t.ok && a.lin1.t.ok && a.lin2.t.ok;
      a.n1_g = upload_tensor(pool, tm.get(q + "norm1.weight"));
      a.n1_b = upload_tensor(pool, tm.get(q + "norm1.bias"));
      a.n2_g = upload_tensor(pool, tm.get(q + "norm2.weight"));
      a.n2_b = upload_tensor(pool, tm.get(q + "norm2.bias"));
    }
  }
  if (f0_gen == SSB_F0_GEN_CONV) {
    // f0_gen 'conv' (stylesinger.py:73-82): FastSpeech2 built pitch_predictor (unused with gmdiff, not packed then) and
    // StyleSinger rebuilds it with the same shapes; pitch_inpainter_predictor is the second one.  No F0 DiffNets.
    PK(build_pitch_predictor(tm, pool, "pitch_predictor.", H, &m->pp[0]));
    PK(build_pitch_predictor(tm, pool, "pitch_inpainter_predictor.", H, &m->pp[1]));
  } else {
    PK(build_denoiser(tm, pool, "gm_diffnet.", hp.f0_channels, hp.f0_layers, hp.f0_cycle, 1, 3, true, &m->f0net[0]));
    PK(build_denoiser(tm, pool, "gm_diffnet_inpainte.", hp.f0_channels, hp.f0_layers, hp.f0_cycle, 1, 3, true, &m->f0net[1]));
  }
  if (prodiff) {
    // StyleSinger.__init__ with decoder 'prodiff' (stylesinger.py:111-117): the mel DiffNet is diff_decoder.denoise_fn; there
    // is no postdiff / ln_proj, and mel_out (built by FastSpeech2.__init__) is not used at inference (:176-177)
    PK(build_denoiser(tm, pool, "diff_decoder.denoise_fn.", hp.mel_channels, hp.mel_layers, hp.mel_cycle, hp.mel_bins, hp.mel_bins, false, &m->melnet));
  } else if (fft) {
    // decoder 'fft' (stylesinger.py:185-186): run_decoder = mel_out(decoder(x)) * tgt_nonpadding; no ln_proj / postdiff
    PK(pack_linear(pool, tm.get("mel_out.weight"), tm.get("mel_out.bias"), &m->mel_out));
  } else {
    PK(build_denoiser(tm, pool, "postdiff.denoise_fn.", hp.mel_channels, hp.mel_layers, hp.mel_cycle, hp.mel_bins, hp.mel_bins, false, &m->melnet));
    PK(pack_linear(pool, tm.get("mel_out.weight"), tm.get("mel_out.bias"), &m->mel_out));
    PK(pack_linear(pool, tm.get("ln_proj.weight", {H, m->cond_width}), tm.get("ln_proj.bias"), &m->ln_proj));
  }
  m->log_eps = logf(1e-30f);
  if (cudaStreamCreateWithFlags(&m->aux_stream, cudaStreamNonBlocking) != cudaSuccess) m->aux_stream = nullptr;
  if (m->aux_stream && (cudaEventCreateWithFlags(&m->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
                        cudaEventCreateWithFlags(&m->ev_join, cudaEventDisableTiming) != cudaSuccess)) {
    cudaStreamDestroy(m->aux_stream);
    m->aux_stream = nullptr;
  }
  if (!tm.missing.empty()) goto fail;
  SSB_CUDA(cudaDeviceSynchronize());
  return 0;
fail:
  if (!tm.missing.empty()) set_error("ssb_model_create: " + tm.missing);
  return -1;
}

int build_vocoder(TensorMap& tm, const ssb_vocoder_config_ex& cfg, Vocoder* v) {
  DevicePool& pool = v->pool;
  v->cfg = cfg;
  v->nk = cfg.n_res;
  v->resblock = cfg.resblock;
  v->nsf = cfg.use_pitch_embed != 0;
  SSB_CHECK(cfg.n_up >= 1 && cfg.n_up <= 8 && cfg.n_res >= 1 && cfg.n_res <= 4, "vocoder: unsupported config");
  SSB_CHECK(cfg.resblock == 1 || cfg.resblock == 2, "vocoder: resblock must be 1 or 2");
  PK(pack_conv(pool, tm.get("conv_pre.weight_v"), tm.get("conv_pre.bias"), 1, PACK_PLAIN, &v->pre, tm.get("conv_pre.weight_g")));
  v->stages.resize(cfg.n_up);
  {
    int rate_after = 1;
    for (int i = 0; i < cfg.n_up; ++i) rate_after *= cfg.up_rates[i];
    int c = cfg.initial_channel;
    int prod_after = rate_after;
    for (int i = 0; i < cfg.n_up; ++i) {
      VocStage& s = v->stages[i];
      const std::string u = "ups." + std::to_string(i) + ".";
      s.u = cfg.up_rates[i];
      s.Cout = c / 2;
      SSB_CHECK(cfg.up_kernels[i] == 2 * cfg.up_rates[i] || cfg.up_kernels[i] - cfg.up_rates[i] >= 0, "vocoder: bad upsample kernel");
      PK(pack_conv_transpose(pool, tm.get(u + "weight_v"), tm.get(u + "weight_g"), tm.get(u + "bias"), s.u, &s.up.f));
      PK(pack_conv_transpose_tc(pool, tm.get(u + "weight_v"), tm.get(u + "weight_g"), s.u, s.up.f.bias, &s.up.t));
      prod_after /= s.u;
      if (v->nsf) {
        const std::string n = "noise_convs." + std::to_string(i) + ".";
        s.nc_s = prod_after;  // stride = prod(upsample_rates[i+1:]) (hifigan_nsf.py:126-132)
        s.nc_w = upload_tensor(pool, tm.get(n + "weight"));
        s.nc_b = upload_tensor(pool, tm.get(n + "bias"));
        if (const HostTensor* wt = tm.get(n + "weight")) {  // [C, 1, K] -> [K, C]: lanes of the tiled kernel read contiguous channels
          const int K = s.nc_s == 1 ? 1 : 2 * s.nc_s, Cn = s.Cout;
          if (wt->numel() == (size_t)K * Cn) {
            std::vector<float> T((size_t)K * Cn);
            for (int cc = 0; cc < Cn; ++cc)
              for (int j = 0; j < K; ++j) T[(size_t)j * Cn + cc] = wt->data[(size_t)cc * K + j];
            s.nc_wt = pool.upload(T);
          }
        }
      }
      // C = 32, 16, 8: time-grouped packing (pack_conv_grouped).  At C = 32 the FFMA GEMM runs the convs as they are and
      // only the tensor-core packing is grouped; at C = 16 and 8 both are (ssb_vocoder_create_ex checked the stage rate).
      const int G = s.Cout < 64 && 64 % s.Cout == 0 ? 64 / s.Cout : 1;
      s.g = G;
      s.res_tc = true;
      const int nconv = cfg.resblock == 1 ? 3 : 2;
      for (int j = 0; j < cfg.n_res; ++j) {
        for (int mI = 0; mI < nconv; ++mI) {
          // ResBlock1 (hifigan_nsf.py:30-66): convs1.{m} at dilation d[m], then convs2.{m} at 1; ResBlock2 (:69-90): convs.{m}
          const std::string q = "resblocks." + std::to_string(i * cfg.n_res + j) + ".";
          struct { std::string p; int dil; Dense* d; } cv[2];
          int ncv = 0;
          if (cfg.resblock == 1) {
            cv[ncv++] = {q + "convs1." + std::to_string(mI) + ".", cfg.res_dilations[j][mI], &s.rb[j].c1[mI]};
            cv[ncv++] = {q + "convs2." + std::to_string(mI) + ".", 1, &s.rb[j].c2[mI]};
          } else {
            cv[ncv++] = {q + "convs." + std::to_string(mI) + ".", cfg.res_dilations[j][mI], &s.rb[j].c1[mI]};
          }
          if (G <= 2) {  // the ungrouped packing (C = 32: the FFMA path's)
            for (int x = 0; x < ncv; ++x)
              PK(pack_dense(pool, tm.get(cv[x].p + "weight_v"), tm.get(cv[x].p + "bias"), cv[x].dil, PACK_PLAIN, cv[x].d,
                            tm.get(cv[x].p + "weight_g")));
            if (G == 1)
              for (int x = 0; x < ncv; ++x)
                if (!cv[x].d->t.ok) s.res_tc = false;
          }
          if (G > 1) {
            for (int x = 0; x < ncv; ++x) {
              const HostTensor* b = tm.get(cv[x].p + "bias");
              PK(pack_conv_grouped(pool, tm.get(cv[x].p + "weight_v"), tm.get(cv[x].p + "weight_g"), cv[x].dil, G,
                                   b ? b->data : nullptr, G > 2, cv[x].d));
              if (!cv[x].d->t.ok) s.res_tc = false;
            }
          }
        }
      }
      c /= 2;
    }
  }
  // conv_post runs on conv_post_tanh (C % 4 == 0): no conv_gemm Cin % 16 rule, so V2's 8-channel last stage packs too
  PK(pack_conv_impl(pool, tm.get("conv_post.weight_v"), tm.get("conv_post.bias"), 1, PACK_PLAIN, &v->post,
                    tm.get("conv_post.weight_g"), false));
  if (v->nsf) {
    v->lin_w = upload_tensor(pool, tm.get("m_source.l_linear.weight", {1, 9}));
    v->lin_b = upload_tensor(pool, tm.get("m_source.l_linear.bias", {1}));
  }
  if (!tm.missing.empty()) goto fail;
  SSB_CUDA(cudaDeviceSynchronize());
  return 0;
fail:
  if (!tm.missing.empty()) set_error("ssb_vocoder_create: " + tm.missing);
  return -1;
}

// Step-bias table: d[t][l][:] = diffusion_projection_l(mlp(SinusoidalPosEmb(t)))  (net.py:114-115,67)
static int build_dtab(Denoiser& d, DevicePool& pool, int T, const float* step_emb_host, cudaStream_t stream) {
  const int C = d.C, L = d.L;
  Seq s;
  int32_t offs[2] = {0, T};
  s.build(offs, 1);
  const size_t rows = (size_t)s.rows();
  // temporary device scratch
  const size_t ws_bytes = (rows * (size_t)(6 * C + L * C) + 65536) * sizeof(float);
  void* ws = nullptr;
  SSB_CUDA(cudaMalloc(&ws, ws_bytes));
  Ctx ctx;
  ctx.base = (char*)ws; ctx.cap = ws_bytes; ctx.stream = stream;
  int rc = 0;
  SeqDev sd;
  rc = upload_layout(ctx, s, 1, &sd);
  float* e = alloc_rows(ctx, sd, C);
  float* h = alloc_rows(ctx, sd, 4 * C);
  float* o = alloc_rows(ctx, sd, C);
  float* emb_t = nullptr;
  if (rc == 0 && (ctx.failed || !e || !h || !o)) rc = -1;
  if (rc == 0) {
    cudaError_t ce = cudaMalloc((void**)&emb_t, (size_t)T * C * sizeof(float));
    if (ce != cudaSuccess) rc = -2;
  }
  if (rc == 0) {
    cudaMemcpyAsync(emb_t, step_emb_host, (size_t)T * C * sizeof(float), cudaMemcpyHostToDevice, stream);
    rc = pack_rows(ctx, sd, emb_t, C, e, C, C);
  }
  if (rc == 0) {
    ConvGemm g = make_gemm(d.mlp0, sd, e, C);
    g.e.act = ACT_MISH; g.e.out = h; g.e.ldo = 4 * C;
    rc = conv_gemm(ctx, g);
  }
  if (rc == 0) {
    ConvGemm g = make_gemm(d.mlp2, sd, h, 4 * C);
    g.e.out = o; g.e.ldo = C;
    rc = conv_gemm(ctx, g);
  }
  float* dt = nullptr;
  if (rc == 0) {
    dt = pool.alloc((size_t)T * L * C);
    if (!dt) rc = -2;
  }
  float* tmp = nullptr;
  if (rc == 0) {
    tmp = alloc_rows(ctx, sd, L * C);
    if (ctx.failed || !tmp) {
      // scratch too small for the guarded [rows, L*C] buffer: allocate separately
      rc = -1;
    }
  }
  if (rc == 0) {
    for (int l = 0; l < L && rc == 0; ++l) {
      ConvGemm g = make_gemm(d.layers[l].dproj, sd, o, C);
      g.e.out = tmp + (size_t)l * C; g.e.ldo = L * C;
      rc = conv_gemm(ctx, g);
    }
    if (rc == 0) rc = unpack_rows(ctx, sd, tmp, L * C, dt, L * C, L * C);
  }
  cudaStreamSynchronize(stream);
  cudaFree(ws);
  if (emb_t) cudaFree(emb_t);
  if (rc == 0) {
    d.dtab = dt;
    d.T = T;
  } else if (g_err.empty()) {
    set_error("set_schedule: building the step table failed");
  }
  return rc;
}

int set_schedule(Model* m, int which, int T, const float* step_emb, const float* gtab, const float* mtab,
                 cudaStream_t stream) {
  SSB_CHECK(which != 0 || m->mel_decoder != SSB_MEL_DECODER_FFT,
            "set_schedule: a model with the FFT mel decoder (SSB_MEL_DECODER_FFT) has no mel diffusion schedule (which = 0)");
  SSB_CHECK(T >= 1 && T <= 4000, "set_schedule: bad T");
  SSB_CHECK(step_emb && gtab, "set_schedule: null tables");
  std::vector<float> g(gtab, gtab + (size_t)T * 8);
  if (which == 0) {
    Denoiser& d = m->melnet;
    float *old_d = d.dtab, *old_g = d.gtab;  // a T sweep re-sets the schedule: the previous tables are released
    if (build_dtab(d, m->pool, T, step_emb, stream)) return -1;
    d.gtab = m->pool.upload(g);
    d.gtab_h = g;
    m->pool.release(old_d);
    m->pool.release(old_g);
  } else {
    SSB_CHECK(m->f0_gen == SSB_F0_GEN_GMDIFF,
              "set_schedule: a model with the conv F0 generator (SSB_F0_GEN_CONV) has no F0 diffusion schedule (which = 1)");
    SSB_CHECK(mtab != nullptr, "set_schedule: multinomial table required for the F0 nets");
    std::vector<float> mt(mtab, mtab + (size_t)T * 8);
    for (int i = 0; i < 2; ++i) {
      Denoiser& d = m->f0net[i];
      float *old_d = d.dtab, *old_g = d.gtab, *old_m = d.mtab;
      if (build_dtab(d, m->pool, T, step_emb, stream)) return -1;
      d.gtab = m->pool.upload(g);
      d.mtab = m->pool.upload(mt);
      d.gtab_h = g;
      m->pool.release(old_d);
      m->pool.release(old_g);
      m->pool.release(old_m);
    }
  }
  SSB_CUDA(cudaStreamSynchronize(stream));
  return 0;
}

}  // namespace ssb
