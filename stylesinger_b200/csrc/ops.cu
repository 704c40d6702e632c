// HBM-bound operators (see ops.cuh).  Thread mapping: blockDim = (32, 8): x over channels, y over rows;
// grid = (ceil(maxlen / 8), B).  Loads along the channel axis are contiguous (coalesced).
#include "ops.cuh"
#include "philox.cuh"

namespace ssb {

namespace {

constexpr int RPB = 8;  // rows per block

inline dim3 row_grid(const SeqDev& s, int rows_per_block = RPB) {
  return dim3((unsigned)((s.maxlen + rows_per_block - 1) / rows_per_block), (unsigned)s.B);
}
#define ROW_SETUP()                                   \
  const int b = blockIdx.y;                           \
  const int4 u = utt[b];                              \
  const int t = blockIdx.x * blockDim.y + threadIdx.y;\
  if (t >= u.y) return;                               \
  const int64_t r = (int64_t)u.x + t;                 \
  const int64_t ti = (int64_t)u.z + t;                \
  (void)ti; (void)r;

// ------------------------------------------------------------------------------------------------
__global__ void k_pack(const int4* utt, const float* tight, int ld_t, float* g, int ld_g, int C, int dir) {
  ROW_SETUP();
  for (int c = threadIdx.x; c < C; c += 32) {
    if (dir == 0) g[r * ld_g + c] = tight[ti * ld_t + c];
    else const_cast<float*>(tight)[ti * ld_t + c] = g[r * ld_g + c];
  }
}
__global__ void k_pack_i32(const int4* utt, const int32_t* tight, int32_t* g, int dir) {
  ROW_SETUP();
  if (threadIdx.x == 0) {
    if (dir == 0) g[r] = tight[ti];
    else const_cast<int32_t*>(tight)[ti] = g[r];
  }
}
__global__ void k_unpack_col_i32(const int4* utt, const int32_t* g, int ld, int col, int32_t* tight) {
  ROW_SETUP();
  if (threadIdx.x == 0) tight[ti * ld + col] = g[r * ld + col];
}
__global__ void k_fill(const int4* utt, float* x, int ld, int C, float v) {
  ROW_SETUP();
  for (int c = threadIdx.x; c < C; c += 32) x[r * ld + c] = v;
}

// one warp per row (threadIdx.x = lane)
__global__ void k_layernorm(const int4* utt, const float* x, int ldx, float* y, int ldy, int C, const float* gamma,
                            const float* beta, float eps, const float* rowmask) {
  ROW_SETUP();
  const float* xr = x + r * ldx;
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += 32) s += xr[c];
  const float mean = warp_sum(s) / (float)C;
  float v = 0.f;
  for (int c = threadIdx.x; c < C; c += 32) {
    const float d = xr[c] - mean;
    v += d * d;
  }
  const float rstd = rsqrtf(warp_sum(v) / (float)C + eps);
  const float m = rowmask ? rowmask[r] : 1.0f;
  for (int c = threadIdx.x; c < C; c += 32) y[r * ldy + c] = ((xr[c] - mean) * rstd * gamma[c] + beta[c]) * m;
}

__global__ void k_row_nonzero(const int4* utt, const float* x, int ld, int C, float* mask) {
  ROW_SETUP();
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += 32) s += fabsf(x[r * ld + c]);
  s = warp_sum(s);
  if (threadIdx.x == 0) mask[r] = s > 0.f ? 1.f : 0.f;
}
__global__ void k_col0_nonzero(const int4* utt, const float* x, int ld, float* mask) {
  ROW_SETUP();
  if (threadIdx.x == 0) mask[r] = x[r * ld] != 0.f ? 1.f : 0.f;
}
__global__ void k_tok_nonzero(const int4* utt, const int32_t* tok, float* mask) {
  ROW_SETUP();
  if (threadIdx.x == 0) mask[r] = tok[r] != 0 ? 1.f : 0.f;
}
// one warp per utterance: sequential ballot scan
__global__ void k_positions(const int4* utt, int B, const float* mask, int32_t* pos) {
  const int b = blockIdx.x;
  if (b >= B) return;
  const int4 u = utt[b];
  int run = 0;
  for (int t0 = 0; t0 < u.y; t0 += 32) {
    const int t = t0 + threadIdx.x;
    const bool on = t < u.y && mask[(int64_t)u.x + t] != 0.f;
    const unsigned bal = __ballot_sync(0xffffffffu, on);
    const int incl = run + __popc(bal & (0xffffffffu >> (31 - threadIdx.x)));
    if (t < u.y) pos[(int64_t)u.x + t] = on ? incl : 0;
    run += __popc(bal);
  }
}
__global__ void k_add_positional(const int4* utt, float* x, int ld, int C, const int32_t* pos, const float* table,
                                 int table_rows, const float* alpha_ptr) {
  ROW_SETUP();
  const float a = alpha_ptr ? alpha_ptr[0] : 1.0f;
  int p = pos[r];
  if (p >= table_rows) p = table_rows - 1;  // host sizes the table so this never triggers
  for (int c = threadIdx.x; c < C; c += 32) x[r * ld + c] += a * table[(int64_t)p * C + c];
}

__global__ void k_embed(const int4* utt, const int32_t* idx, const float* table, int nt, float scale, float* x, int ld,
                        int C, int accumulate) {
  ROW_SETUP();
  int i = idx[r];
  i = i < 0 ? 0 : (i >= nt ? nt - 1 : i);
  for (int c = threadIdx.x; c < C; c += 32) {
    const float v = scale * table[(int64_t)i * C + c];
    x[r * ld + c] = accumulate ? x[r * ld + c] + v : v;
  }
}
__global__ void k_note_encoder(const int4* utt, const int32_t* note, const int32_t* type, const float* dur,
                               const float* En, const float* Et, const float* w, const float* bb, float scale, float* x,
                               int ld, int C, int accumulate) {
  ROW_SETUP();
  int n = note[r], ty = type[r];
  n = n < 0 ? 0 : (n > 99 ? 99 : n);
  ty = ty < 0 ? 0 : (ty > 4 ? 4 : ty);
  const float d = dur[r];
  for (int c = threadIdx.x; c < C; c += 32) {
    // reference order: x = emb*16 ; x = x + durs + types   (stylesinger.py:32-35)
    float v = En[n * C + c] * scale;
    v = v + (d * w[c] + bb[c]);
    v = v + Et[ty * C + c] * scale;
    x[r * ld + c] = accumulate ? x[r * ld + c] + v : v;
  }
}
__global__ void k_expand(const int4* utt, const int4* utt_ph, const int32_t* mel2ph, const float* src, int ld_s,
                         float* out, int ld_o, int C, const int32_t* note, int32_t* midi, float* tgt_nonpad) {
  ROW_SETUP();
  const int4 up = utt_ph[b];
  int m = mel2ph[r];
  if (m < 0 || m > up.y) m = 0;
  const int64_t rs = (int64_t)up.x + m - 1;
  for (int c = threadIdx.x; c < C; c += 32) out[r * ld_o + c] = m > 0 ? src[rs * ld_s + c] : 0.f;
  if (threadIdx.x == 0) {
    if (midi) midi[r] = m > 0 ? note[rs] : 0;
    if (tgt_nonpad) tgt_nonpad[r] = m > 0 ? 1.f : 0.f;
  }
}
__global__ void k_combine(const int4* utt, CombineArgs a) {
  ROW_SETUP();
  const float m = a.rowmask ? a.rowmask[r] : 1.f;
  for (int c = threadIdx.x; c < a.C; c += 32) {
    float v = a.m[0][r * a.ldm[0] + c];
#pragma unroll
    for (int i = 1; i < 4; ++i)
      if (a.m[i]) v += a.m[i][r * a.ldm[i] + c];
#pragma unroll
    for (int i = 0; i < 3; ++i)
      if (a.v[i]) v += a.v[i][(int64_t)b * a.C + c];
    a.out[r * a.ldo + c] = v * m;
  }
}

__global__ void k_smar(const int4* utt, const float* x, int ldx, int C, const float* mask, const float* rs, float* y, int ldy) {
  ROW_SETUP();
  const float m = mask[r], a = rs ? rs[r] : 0.f;
  for (int c = threadIdx.x; c < C; c += 32) y[r * ldy + c] = x[r * ldx + c] * m + a;
}
__global__ void k_concat2_pos(const int4* utt, const float* z, int C, const int32_t* pos, const float* table,
                              int table_rows, float* out, int ldo) {
  ROW_SETUP();
  int p = pos[r];
  if (p >= table_rows) p = table_rows - 1;
  for (int c = threadIdx.x; c < C; c += 32) {
    out[r * ldo + c] = z[r * C + c];
    out[r * ldo + C + c] = table[(int64_t)p * C + c];
  }
}
__global__ void k_concat_cond(const int4* utt, const float* coarse, const float* dec, const float* spk, const float* emo,
                              const float* style, float* out, int ldo) {
  ROW_SETUP();
  float* o = out + r * ldo;
  for (int c = threadIdx.x; c < 80; c += 32) o[c] = coarse[r * 80 + c];
  // the 256-column segments that are present, in the reference's order; dec / emo / style may be null
  const int o_dec = 80, o_spk = o_dec + (dec ? 256 : 0), o_emo = o_spk + 256, o_sty = o_emo + (emo ? 256 : 0);
  for (int c = threadIdx.x; c < 256; c += 32) {
    if (dec) o[o_dec + c] = dec[r * 256 + c];
    o[o_spk + c] = spk[(int64_t)b * 256 + c];
    if (emo) o[o_emo + c] = emo[(int64_t)b * 256 + c];
    if (style) o[o_sty + c] = style[r * 256 + c];
  }
}
__global__ void k_clip(const int4* utt, float* x, int ld, int C, float lo, float hi) {
  ROW_SETUP();
  for (int c = threadIdx.x; c < C; c += 32) x[r * ld + c] = fminf(fmaxf(x[r * ld + c], lo), hi);
}

__global__ void k_dur(const int4* utt, const float* logdur, const float* nonpad, int32_t* dur) {
  ROW_SETUP();
  if (threadIdx.x == 0) {
    float d = rintf(expf(logdur[r]) - 1.0f);  // torch.round = round-half-even = rintf
    d = fmaxf(d, 0.f);
    dur[r] = nonpad[r] != 0.f ? (int32_t)d : 0;
  }
}
// one block per utterance; frames of the utterance search the cumulative durations
__global__ void k_length_regulate(const int4* utt_f, const int4* utt_p, const int32_t* dur, int32_t* mel2ph) {
  const int b = blockIdx.x;
  const int4 uf = utt_f[b], up = utt_p[b];
  extern __shared__ int cs[];  // inclusive cumsum, up.y entries
  if (threadIdx.x == 0) {
    int run = 0;
    for (int p = 0; p < up.y; ++p) {
      run += dur[(int64_t)up.x + p];
      cs[p] = run;
    }
  }
  __syncthreads();
  for (int f = threadIdx.x; f < uf.y; f += blockDim.x) {
    int lo = 0, hi = up.y;  // first p with cs[p] > f
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (cs[mid] > f) hi = mid; else lo = mid + 1;
    }
    mel2ph[(int64_t)uf.x + f] = lo < up.y ? lo + 1 : 0;
  }
}

// ------------------------------------------------------------------------------------------------
// RVQ: one warp per row, D = 256 (8 values per lane).  dist = (|x|^2 + |c|^2) - 2 x.c  in fp32 with the
// reference's association (RQ.py:39-46); argmin ties -> lowest index.
__global__ void k_cb_norm(const float* cb, int n, float* out) {
  const int i = blockIdx.x * blockDim.y + threadIdx.y;
  if (i >= n) return;
  float s = 0.f;
  for (int c = threadIdx.x; c < 256; c += 32) {
    const float v = cb[(int64_t)i * 256 + c];
    s += v * v;
  }
  s = warp_sum(s);
  if (threadIdx.x == 0) out[i] = s;
}
__global__ void k_rvq(const int4* utt, const float* x, int ldx, const float* cb, const float* cbn, int n_embed, int depth,
                      float* quant, int ldq, int32_t* codes) {
  ROW_SETUP();
  const int lane = threadIdx.x;
  float xv[8], res[8], agg[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    xv[i] = x[r * ldx + lane + 32 * i];
    res[i] = xv[i];
    agg[i] = 0.f;
  }
  for (int d = 0; d < depth; ++d) {
    float n2 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) n2 += res[i] * res[i];
    n2 = warp_sum(n2);
    const float* cbd = cb + (int64_t)d * n_embed * 256;
    float best = INFINITY;
    int besti = 0;
    for (int e = 0; e < n_embed; ++e) {
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) dot = fmaf(res[i], cbd[(int64_t)e * 256 + lane + 32 * i], dot);
      dot = warp_sum(dot);
      const float dist = (n2 + cbn[d * n_embed + e]) + (-2.0f) * dot;
      if (dist < best) { best = dist; besti = e; }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float q = cbd[(int64_t)besti * 256 + lane + 32 * i];
      res[i] -= q;
      agg[i] += q;
    }
    if (lane == 0) codes[r * depth + d] = besti;
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) quant[r * ldq + lane + 32 * i] = xv[i] + (agg[i] - xv[i]);
}

// ------------------------------------------------------------------------------------------------
// samplers
// Injected noise is indexed by the tight row ti of the call; a Philox draw by the utterance's counter row g.row0 + t under
// its key g.key (SeqDev::rng).  `per` draws per row, element j of the row.
__device__ __forceinline__ float noise_n(const float* noise, int64_t ti, const UttRng& g, int t, int per, int j,
                                         uint64_t stream_id) {
  return noise ? noise[ti * per + j] : philox_normal(g.key, stream_id, (uint64_t)((int64_t)g.row0 + t) * per + j);
}
__device__ __forceinline__ float noise_u(const float* noise, int64_t ti, const UttRng& g, int t, int per, int j,
                                         uint64_t stream_id) {
  return noise ? noise[ti * per + j] : philox_uniform(g.key, stream_id, (uint64_t)((int64_t)g.row0 + t) * per + j);
}

__global__ void k_mel_q_sample(const int4* utt, const UttRng* rng, const float* coarse, int ldc, const float* noise,
                               const float* smin, const float* smax, float sa, float s1a, float* x, int ldx, uint64_t sid) {
  ROW_SETUP();
  const UttRng g = rng[b];
  for (int c = threadIdx.x; c < 80; c += 32) {
    if (!coarse) {  // ProDiff: x_T = randn, no coarse mel and no normalisation (prodiff.py:214-216)
      x[r * ldx + c] = noise_n(noise, ti, g, t, 80, c, sid);
      continue;
    }
    const float x0 = (coarse[r * ldc + c] - smin[c]) / (smax[c] - smin[c]) * 2.0f - 1.0f;
    x[r * ldx + c] = sa * x0 + s1a * noise_n(noise, ti, g, t, 80, c, sid);
  }
}
// DDPM (shallow_diffusion_tts.py:145-162): eps -> clipped x0.  ProDiff (prodiff.py:135-148): the table holds (0, -1) in
// slots 0-1 so x0 = eps exactly, and clip = 0.
__global__ void k_mel_p_sample(const int4* utt, const UttRng* rng, float* x, int ldx, const float* eps, int lde,
                               const float* noise, const float* tab, uint64_t sid, int clip) {
  ROW_SETUP();
  const UttRng g = rng[b];
  const float a = tab[0], bq = tab[1], c1 = tab[2], c2 = tab[3], sig = tab[4];
  for (int c = threadIdx.x; c < 80; c += 32) {
    const float xt = x[r * ldx + c];
    float x0 = a * xt - bq * eps[r * lde + c];
    if (clip) x0 = fminf(fmaxf(x0, -1.0f), 1.0f);
    const float mean = c1 * x0 + c2 * xt;
    // reference: mean + nonzero_mask * exp(0.5*logvar) * noise ; sig already folds the mask
    x[r * ldx + c] = mean + sig * noise_n(noise, ti, g, t, 80, c, sid);
  }
}
// PLMS update (shallow_diffusion_tts.py:164-197).  prime = (w0*eps + w1*h1 + w2*h2 + w3*h3) / den; x_out = x + x_delta with
//   x_delta = (a_prev - a_t) * (x / (sqrt(a_t) * (sqrt(a_t) + sqrt(a_prev)))
//                               - prime / (sqrt(a_t) * (sqrt((1 - a_prev) * a_t) + sqrt((1 - a_t) * a_prev))))     (get_x_pred)
// and, when hist_out is given, hist_out <- eps (the un-extrapolated prediction joins the history, :194).
__global__ void k_plms_update(const int4* utt, PlmsArgs a) {
  ROW_SETUP();
  const float a_t = a.a_t, a_prev = a.a_prev;
  const float a_t_sq = sqrtf(a_t), a_prev_sq = sqrtf(a_prev);
  const float kx = 1.0f / (a_t_sq * (a_t_sq + a_prev_sq));
  const float ke = 1.0f / (a_t_sq * (sqrtf((1.0f - a_prev) * a_t) + sqrtf((1.0f - a_t) * a_prev)));
  const float da = a_prev - a_t;
  for (int c = threadIdx.x; c < 80; c += 32) {
    const float e = a.eps[r * a.lde + c];
    float pr = a.w0 * e;
    if (a.h1) pr += a.w1 * a.h1[r * 80 + c];
    if (a.h2) pr += a.w2 * a.h2[r * 80 + c];
    if (a.h3) pr += a.w3 * a.h3[r * 80 + c];
    pr = pr / a.den;
    const float xt = a.x[r * 80 + c];
    a.x_out[r * 80 + c] = xt + da * (kx * xt - ke * pr);
    if (a.hist_out) a.hist_out[r * 80 + c] = e;
  }
}
__global__ void k_mel_denorm(const int4* utt, const float* x, int ldx, const float* smin, const float* smax,
                             const float* rowmask, float* mel, int ld) {
  ROW_SETUP();
  const float m = rowmask ? rowmask[r] : 1.f;
  for (int c = threadIdx.x; c < 80; c += 32)
    mel[ti * ld + c] = ((x[r * ldx + c] + 1.0f) / 2.0f * (smax[c] - smin[c]) + smin[c]) * m;
}

__device__ __forceinline__ float log_add_exp(float a, float b) {
  const float m = fmaxf(a, b);
  return m + logf(expf(a - m) + expf(b - m));
}
__global__ void k_f0_init(const int4* utt, const UttRng* rng, float* z, int32_t* uv, const float* gnoise, uint64_t sid) {
  ROW_SETUP();
  if (threadIdx.x == 0) {
    z[r] = noise_n(gnoise, ti, rng[b], t, 1, 0, sid);
    uv[r] = 0;  // log_sample_categorical over a size-1 class dim (gaussian_multinomial_diffusion.py:924-926)
  }
}
__global__ void k_f0_p_sample(const int4* utt, F0StepArgs a) {
  ROW_SETUP();
  if (threadIdx.x != 0) return;
  const UttRng g = a.rng[b];
  const float ln2 = 0.69314718055994530942f;
  const float* o = a.out3 + r * a.ld3;
  // gaussian half (gaussian_p_sample, :325-333)
  const float zt = a.z[r];
  float x0 = a.gtab[0] * zt - a.gtab[1] * o[0];
  x0 = fmaxf(fminf(x0, a.hi[r]), a.lo[r]);
  const float mean = a.gtab[2] * x0 + a.gtab[3] * zt;
  a.z[r] = mean + a.gtab[4] * noise_n(a.gnoise, ti, g, t, 1, 0, a.gauss_stream);
  // multinomial half (p_pred / q_posterior, :374-413)
  const float l0a = o[1], l0b = o[2];
  const float mx = fmaxf(l0a, l0b);
  const float lse = mx + logf(expf(l0a - mx) + expf(l0b - mx));
  const float ls0 = l0a - lse, ls1 = l0b - lse;  // log_softmax
  float e0, e1;
  if (a.t == 0) { e0 = ls0; e1 = ls1; }
  else {
    e0 = log_add_exp(ls0 + a.mtab[2], a.mtab[3] - ln2);
    e1 = log_add_exp(ls1 + a.mtab[2], a.mtab[3] - ln2);
  }
  const int cur = a.uv[r];
  const float lz0 = cur == 0 ? 0.f : a.log_eps, lz1 = cur == 1 ? 0.f : a.log_eps;
  const float u0 = e0 + log_add_exp(lz0 + a.mtab[0], a.mtab[1] - ln2);
  const float u1 = e1 + log_add_exp(lz1 + a.mtab[0], a.mtab[1] - ln2);
  const float m2 = fmaxf(u0, u1);
  const float lse2 = m2 + logf(expf(u0 - m2) + expf(u1 - m2));  // torch.logsumexp
  const float p0 = u0 - lse2, p1 = u1 - lse2;
  const float r0 = noise_u(a.unoise, ti, g, t, 2, 0, a.unif_stream);
  const float r1 = noise_u(a.unoise, ti, g, t, 2, 1, a.unif_stream);
  const float g0 = -logf(-logf(r0 + 1e-30f) + 1e-30f);
  const float g1 = -logf(-logf(r1 + 1e-30f) + 1e-30f);
  a.uv[r] = (g1 + p1) > (g0 + p0) ? 1 : 0;  // argmax, ties -> 0
}
__global__ void k_ddiff_input(const int4* utt, const float* z, const int32_t* uv, const float* w, const float* bb,
                              const float* Euv, const float* d0, float* x, float* y, int C, __half* yh, __half* yl) {
  ROW_SETUP();
  const int h = C / 2;
  const float f = z[r];
  const int cls = uv[r];
  for (int c = threadIdx.x; c < C; c += 32) {
    const float v = c < h ? (f * w[c] + bb[c]) : Euv[cls * h + (c - h)];
    if (x) x[r * C + c] = v;
    const float yy = v + d0[c];
    if (y) y[r * C + c] = yy;
    if (yh) {
      const __half h = __float2half_rn(yy);
      yh[r * C + c] = h;
      yl[r * C + c] = __float2half_rn(yy - __half2float(h));
    }
  }
}

// pitch glue
__device__ __forceinline__ float minmax_norm_(float x) {
  x = fminf(x, 10.0f);
  return (x - 6.0f) / (10.0f - 6.0f) * 2.0f - 1.0f;
}
__global__ void k_midi_band(const int4* utt, const int32_t* midi, float* lo, float* hi) {
  ROW_SETUP();
  if (threadIdx.x != 0) return;
  const float m = (float)midi[r];
  // (2 ** ((m +- 3 - 69) / 12) * 440).log2()   (stylesinger.py:276-279)
  const float up = log2f(exp2f((m + 3.0f - 69.0f) / 12.0f) * 440.0f);
  const float dn = log2f(exp2f((m - 3.0f - 69.0f) / 12.0f) * 440.0f);
  hi[r] = fminf(fmaxf(minmax_norm_(up), -1.f), 1.f);
  lo[r] = fminf(fmaxf(minmax_norm_(dn), -1.f), 1.f);
}
// The tail of inpaint_pitch shared by both F0 generators (stylesinger.py:237-243): f0 (log2 Hz) and uv of row r ->
// f0_denorm (Hz) and the coarse pitch bin.
__device__ __forceinline__ void f0_denorm_coarse(float f0, bool uv, int32_t mel2ph, float* f0_denorm, int32_t* pitch) {
  float hz = exp2f(f0);  // denorm_f0, pitch_norm == 'log' (utils/pitch_utils.py:65-78)
  if (uv) hz = 0.f;
  if (mel2ph == 0) hz = 0.f;
  *f0_denorm = hz;
  // f0_to_coarse (utils/pitch_utils.py:22-31)
  const float mel_min = 1127.0f * logf(1.0f + 50.0f / 700.0f);
  const float mel_max = 1127.0f * logf(1.0f + 1100.0f / 700.0f);
  float mel = 1127.0f * logf(1.0f + hz / 700.0f);
  if (mel > 0.f) mel = (mel - mel_min) * 254.0f / (mel_max - mel_min) + 1.0f;
  if (mel <= 1.f) mel = 1.f;
  if (mel > 255.f) mel = 255.f;
  *pitch = (int32_t)(mel + 0.5f);
}
__global__ void k_pitch_glue(const int4* utt, PitchGlueArgs a) {
  ROW_SETUP();
  if (threadIdx.x != 0) return;
  const bool rest = a.midi[r] == 0;
  // add_gmdiff_pitch: uv[midi==0] = 1 ; f0 = minmax_denorm(f0)   (stylesinger.py:287-296)
  const float uva = rest ? 1.f : (float)a.uva[r], uvs = rest ? 1.f : (float)a.uvs[r];
  const float fa = (a.za[r] + 1.0f) / 2.0f * (10.0f - 6.0f) + 6.0f;
  const float fs = (a.zs[r] + 1.0f) / 2.0f * (10.0f - 6.0f) + 6.0f;
  const float pf = fs / 2.0f + fa / 2.0f;  // pitch_domain_specific/2 + pitch_domain_agnostic/2  (:230)
  const float pu = uvs / 2.0f + uva / 2.0f;
  if (a.pitch_pred) { a.pitch_pred[r * 2] = pf; a.pitch_pred[r * 2 + 1] = pu; }
  float f0 = a.f0_in ? a.f0_in[r] : pf;
  const bool uv = a.f0_in ? (a.uv_in ? a.uv_in[r] > 0.f : false) : (pu > 0.f);
  f0_denorm_coarse(f0, uv, a.mel2ph[r], &a.f0_denorm[r], &a.pitch[r]);
}
// f0_gen 'conv' (stylesinger.py:223-236): the two PitchPredictor outputs are averaged as they are - no minmax_denorm, no
// forced-unvoiced rests; uv thresholds the averaged logit.
__global__ void k_pitch_glue_conv(const int4* utt, PitchGlueConvArgs a) {
  ROW_SETUP();
  if (threadIdx.x != 0) return;
  const float pf = a.ps[r * 2] / 2.0f + a.pa[r * 2] / 2.0f;  // pitch_domain_specific/2 + pitch_domain_agnostic/2  (:230)
  const float pu = a.ps[r * 2 + 1] / 2.0f + a.pa[r * 2 + 1] / 2.0f;
  if (a.pitch_pred) { a.pitch_pred[r * 2] = pf; a.pitch_pred[r * 2 + 1] = pu; }
  const float f0 = a.f0_in ? a.f0_in[r] : pf;
  const bool uv = a.f0_in ? (a.uv_in ? a.uv_in[r] > 0.f : false) : (pu > 0.f);
  f0_denorm_coarse(f0, uv, a.mel2ph[r], &a.f0_denorm[r], &a.pitch[r]);
}

// ------------------------------------------------------------------------------------------------
// NSF source (SineGen second definition, source.py:348-441).  Per (utterance, harmonic): two running sums
// accumulated in double and rounded to fp32 per element, like torch's CPU cumsum.
// One block (256 threads) per (utterance, harmonic); chunked block scan with a double carry.
__device__ double block_scan_incl(double v, double* sh, double& total) {
  // blockDim.x == 256; returns inclusive scan of v across the block, total = block sum
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double n = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += n;
  }
  if (lane == 31) sh[w] = v;
  __syncthreads();
  if (w == 0) {
    double s = lane < 8 ? sh[lane] : 0.0;
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) {
      const double n = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += n;
    }
    if (lane < 8) sh[8 + lane] = s;
  }
  __syncthreads();
  const double base = w > 0 ? sh[8 + w - 1] : 0.0;
  total = sh[15];
  __syncthreads();
  return v + base;
}

__global__ void k_nsf_phase(const int4* utt1, const int4* utt256, const UttRng* rng1, const float* f0, const float* rand_ini,
                            float* sines, int upp, float sr) {
  // sines: tight [total256, 9] -> sin(2*pi*phase) (amplitude / uv / noise applied in k_nsf_merge)
  const int b = blockIdx.y, h = blockIdx.x;  // harmonic h in 0..8
  const int4 u1 = utt1[b], u2 = utt256[b];
  __shared__ double sh[16];
  const int N = u2.y;
  float ini = 0.f;
  if (h > 0) ini = rand_ini ? rand_ini[b * 9 + h] : philox_uniform(rng1[b].key, stream_voc_ini(rng1[b].ini), (uint64_t)h);
  double carry1 = 0.0, carry2 = 0.0;
  float prev_over = 0.f;  // tmp_over_one of the previous sample
  for (int n0 = 0; n0 < N; n0 += 256) {
    const int n = n0 + threadIdx.x;
    float rad = 0.f;
    if (n < N) {
      const float f = f0[(int64_t)u1.x + n / upp] * (float)(h + 1);
      rad = fmodf(f / sr, 1.0f);
      if (n == 0) rad = rad + ini;
    }
    double tot;
    const double c1 = block_scan_incl((double)rad, sh, tot) + carry1;
    carry1 += tot;
    const float s1 = (float)c1;                 // fp32 cumsum value
    const float over = fmodf(s1, 1.0f);          // % 1 (non-negative operands)
    // neighbour's value: shuffle within warp, smem across warps
    __shared__ float sprev[256];
    sprev[threadIdx.x] = over;
    __syncthreads();
    const float po = threadIdx.x > 0 ? sprev[threadIdx.x - 1] : prev_over;
    const float last = sprev[255];
    __syncthreads();
    float shift = 0.f;
    if (n > 0 && n < N && (over - po) < 0.f) shift = -1.0f;
    const float v2 = n < N ? (rad + shift) : 0.f;  // fp32 add as in the reference
    const double c2 = block_scan_incl((double)v2, sh, tot) + carry2;
    carry2 += tot;
    if (n < N) {
      const float ph = (float)c2;
      sines[((int64_t)u2.z + n) * 9 + h] = sinf(ph * 2.0f * 3.14159265358979323846f);
    }
    prev_over = last;
  }
}
__global__ void k_nsf_merge(const int4* utt1, const int4* utt256, const UttRng* rng256, const float* f0, const float* sines,
                            const float* noise, const float* lw, const float* lb, float* har, int upp) {
  const int b = blockIdx.y;
  const int4 u1 = utt1[b], u2 = utt256[b];
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= u2.y) return;
  const UttRng g = rng256[b];
  const float f = f0[(int64_t)u1.x + n / upp];
  const float uv = f > 0.f ? 1.f : 0.f;
  const float namp = uv * 0.003f + (1.0f - uv) * 0.1f / 3.0f;
  float acc = lb[0];
  const int64_t ti = (int64_t)u2.z + n;
#pragma unroll
  for (int h = 0; h < 9; ++h) {
    const float s = sines[ti * 9 + h] * 0.1f;
    const float nz = namp * noise_n(noise, ti, g, n, 9, h, stream_voc_src());
    acc = fmaf(s * uv + nz, lw[h], acc);
  }
  har[(int64_t)u2.x + n] = tanhf(acc);
}

__global__ void k_noise_conv_add(const int4* uttx, const int4* utt256, float* x, int ld, int C, const float* har,
                                 const float* w, const float* bb, int s, __half* ph, __half* pl, float pslope) {
  const int b = blockIdx.y;
  const int4 ux = uttx[b], uh = utt256[b];
  const int t = blockIdx.x * blockDim.y + threadIdx.y;
  if (t >= ux.y) return;
  const int64_t r = (int64_t)ux.x + t;
  const int K = s == 1 ? 1 : 2 * s;
  const int pad = s == 1 ? 0 : s / 2;
  for (int c = threadIdx.x; c < C; c += 32) {
    float acc = bb[c];
    for (int j = 0; j < K; ++j) {
      const int64_t q = (int64_t)t * s - pad + j;
      if (q >= 0 && q < uh.y) acc = fmaf(w[c * K + j], har[(int64_t)uh.x + q], acc);
    }
    const float v = x[r * ld + c] + acc;
    x[r * ld + c] = v;
    if (ph) {  // leaky_relu(v) as fp16 hi/lo planes: the A operand of the tensor-core convs that follow
      const float y = v > 0.f ? v : v * pslope;
      const __half h = __float2half_rn(y);
      ph[r * C + c] = h;
      pl[r * C + c] = __float2half_rn(y - __half2float(h));
    }
  }
}
// Tiled variant (C % 4 == 0, weights as [K, C]): a block owns NC_TR consecutive output rows of one utterance, stages the
// har window they read in shared memory once, and every thread updates 4 channels of one row per step with float4 / 8-byte
// accesses.  The row-per-warp kernel above issued one dependent har load per tap and ran at ~5 % of the HBM roofline.
constexpr int NC_TR = 128;
__global__ void __launch_bounds__(256) k_noise_conv_add_tiled(const int4* uttx, const int4* utt256, float* x, int ld, int C, const float* har,
                                                              const float* wt, const float* bb, int s, __half* ph, __half* pl, float pslope) {
  extern __shared__ float sh_har[];  // [NC_TR * s + K]
  const int b = blockIdx.y;
  const int4 ux = uttx[b], uh = utt256[b];
  const int t0 = blockIdx.x * NC_TR;
  if (t0 >= ux.y) return;
  const int K = s == 1 ? 1 : 2 * s;
  const int pad = s == 1 ? 0 : s / 2;
  const int nrow = min(NC_TR, ux.y - t0);
  const int win = nrow * s + K;
  const int64_t q0 = (int64_t)t0 * s - pad;
  for (int i = threadIdx.x; i < win; i += blockDim.x) {
    const int64_t q = q0 + i;
    sh_har[i] = (q >= 0 && q < uh.y) ? har[(int64_t)uh.x + q] : 0.f;
  }
  __syncthreads();
  const int c4n = C >> 2;
  for (int it = threadIdx.x; it < nrow * c4n; it += blockDim.x) {
    const int tl = it / c4n, c = (it - tl * c4n) << 2;
    float4 acc = *reinterpret_cast<const float4*>(bb + c);
    const float* hw = sh_har + tl * s;
    for (int j = 0; j < K; ++j) {
      const float h = hw[j];
      const float4 w4 = __ldg(reinterpret_cast<const float4*>(wt + (size_t)j * C + c));
      acc.x = fmaf(w4.x, h, acc.x); acc.y = fmaf(w4.y, h, acc.y); acc.z = fmaf(w4.z, h, acc.z); acc.w = fmaf(w4.w, h, acc.w);
    }
    const int64_t r = (int64_t)ux.x + t0 + tl;
    float4* xp = reinterpret_cast<float4*>(x + r * ld + c);
    float4 v = *xp;
    v.x += acc.x; v.y += acc.y; v.z += acc.z; v.w += acc.w;
    *xp = v;
    if (ph) {
      const float y0 = v.x > 0.f ? v.x : v.x * pslope, y1 = v.y > 0.f ? v.y : v.y * pslope;
      const float y2 = v.z > 0.f ? v.z : v.z * pslope, y3 = v.w > 0.f ? v.w : v.w * pslope;
      const __half2 h01 = __floats2half2_rn(y0, y1), h23 = __floats2half2_rn(y2, y3);
      const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
      const __half2 l01 = __floats2half2_rn(y0 - f01.x, y1 - f01.y), l23 = __floats2half2_rn(y2 - f23.x, y3 - f23.y);
      uint2 uh2, ul2;
      uh2.x = *reinterpret_cast<const uint32_t*>(&h01); uh2.y = *reinterpret_cast<const uint32_t*>(&h23);
      ul2.x = *reinterpret_cast<const uint32_t*>(&l01); ul2.y = *reinterpret_cast<const uint32_t*>(&l23);
      *reinterpret_cast<uint2*>(ph + r * C + c) = uh2;
      *reinterpret_cast<uint2*>(pl + r * C + c) = ul2;
    }
  }
}
__global__ void k_tanh_out(const int4* utt, const float* x, int ld, float* wav) {
  const int b = blockIdx.y;
  const int4 u = utt[b];
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= u.y) return;
  wav[(int64_t)u.z + t] = tanhf(x[((int64_t)u.x + t) * ld]);
}
// conv_post + tanh of the HiFi-GAN generator (hifigan_nsf.py:165-167): wav[t] = tanh(b + sum_{j,c} W[j][c] * leaky_relu(x[t + j - center][c])).
// N = 1 makes the implicit-GEMM kernels waste 63/64 of a tile; here a block stages CP_T + taps - 1 rows of leaky_relu(x) in
// shared memory (row pitch C + 1: conflict-free) and every thread reduces the window of one output sample.
constexpr int CP_T = 256;
__global__ void __launch_bounds__(CP_T) k_conv_post_tanh(const int4* utt, const float* x, int ld, int C, int taps, int center, const float* W,
                                                         int npad, const float* bias, float slope, float* wav) {
  extern __shared__ float cp_sm[];  // [(CP_T + taps - 1) * (C + 1)] activations, then [taps * C] weights
  const int b = blockIdx.y;
  const int4 u = utt[b];
  const int t0 = blockIdx.x * CP_T;
  if (t0 >= u.y) return;
  const int pitch = C + 1, nr = CP_T + taps - 1;
  float* sw = cp_sm + nr * pitch;
  for (int i = threadIdx.x; i < taps * C; i += CP_T) sw[i] = W[(size_t)i * npad];
  const int c4n = C >> 2;
  for (int i = threadIdx.x; i < nr * c4n; i += CP_T) {
    const int rl = i / c4n, c = (i - rl * c4n) << 2;
    const int t = t0 + rl - center;  // rows outside the utterance are the zero "same" padding
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t >= 0 && t < u.y) v = *reinterpret_cast<const float4*>(x + ((int64_t)u.x + t) * ld + c);
    float* d = cp_sm + rl * pitch + c;
    d[0] = v.x > 0.f ? v.x : v.x * slope; d[1] = v.y > 0.f ? v.y : v.y * slope;
    d[2] = v.z > 0.f ? v.z : v.z * slope; d[3] = v.w > 0.f ? v.w : v.w * slope;
  }
  __syncthreads();
  const int t = t0 + threadIdx.x;
  if (t >= u.y) return;
  float acc = bias ? bias[0] : 0.f;
  for (int j = 0; j < taps; ++j) {
    const float* xr = cp_sm + (threadIdx.x + j) * pitch;
    const float* wr = sw + j * C;
#pragma unroll 8
    for (int c = 0; c < C; ++c) acc = fmaf(xr[c], wr[c], acc);
  }
  wav[(int64_t)u.z + t] = tanhf(acc);
}

__global__ void k_mel_post(const int4* utt, float* mel, int ld, float* f0, float vmin, float vmax) {
  ROW_SETUP();
  for (int c = threadIdx.x; c < 80; c += 32) mel[r * ld + c] = fminf(fmaxf(mel[r * ld + c], vmin), vmax);
}

__global__ void k_mel_post_flat(float* mel, int64_t n, float vmin, float vmax, int32_t* cnt) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.y + threadIdx.y;
  if (r >= n) return;
  float s = 0.f;
  for (int c = threadIdx.x; c < 80; c += 32) {
    const float v = mel[r * 80 + c];
    s += fabsf(v);
    mel[r * 80 + c] = fminf(fmaxf(v, vmin), vmax);
  }
  s = warp_sum(s);
  if (threadIdx.x == 0 && s > 0.f) atomicAdd(cnt, 1);
}

}  // namespace

int mel_postprocess_flat(cudaStream_t st, float* mel, int64_t n, float vmin, float vmax, int32_t* cnt) {
  SSB_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int32_t), st));
  if (n > 0) {
    k_mel_post_flat<<<(unsigned)((n + 7) / 8), dim3(32, 8), 0, st>>>(mel, n, vmin, vmax, cnt);
    SSB_CUDA(cudaGetLastError());
    ++g_launches;
  }
  return 0;
}

#define LAUNCH_ROWS(kern, s, ...)                                            \
  do {                                                                       \
    if (!ctx.dry && s.B > 0 && s.maxlen > 0) {                               \
      kern<<<row_grid(s), dim3(32, RPB), 0, ctx.stream>>>(s.utt, __VA_ARGS__); \
      SSB_CUDA(cudaGetLastError());                                          \
      ++g_launches;                                                          \
    }                                                                        \
  } while (0)

int pack_rows(Ctx& ctx, const SeqDev& s, const float* tight, int ld_t, float* g, int ld_g, int C) {
  LAUNCH_ROWS(k_pack, s, tight, ld_t, g, ld_g, C, 0);
  return 0;
}
int unpack_rows(Ctx& ctx, const SeqDev& s, const float* g, int ld_g, float* tight, int ld_t, int C) {
  LAUNCH_ROWS(k_pack, s, (const float*)tight, ld_t, const_cast<float*>(g), ld_g, C, 1);
  return 0;
}
int pack_rows_i32(Ctx& ctx, const SeqDev& s, const int32_t* tight, int32_t* g) {
  LAUNCH_ROWS(k_pack_i32, s, tight, g, 0);
  return 0;
}
int unpack_rows_i32(Ctx& ctx, const SeqDev& s, const int32_t* g, int32_t* tight) {
  LAUNCH_ROWS(k_pack_i32, s, (const int32_t*)tight, const_cast<int32_t*>(g), 1);
  return 0;
}
int unpack_cols_i32(Ctx& ctx, const SeqDev& s, const int32_t* g, int ld, int col, int32_t* tight) {
  LAUNCH_ROWS(k_unpack_col_i32, s, g, ld, col, tight);
  return 0;
}
int fill_rows(Ctx& ctx, const SeqDev& s, float* x, int ld, int C, float v) {
  LAUNCH_ROWS(k_fill, s, x, ld, C, v);
  return 0;
}
int layernorm_rows(Ctx& ctx, const SeqDev& s, const float* x, int ldx, float* y, int ldy, int C, const float* gamma,
                   const float* beta, float eps, const float* rowmask) {
  LAUNCH_ROWS(k_layernorm, s, x, ldx, y, ldy, C, gamma, beta, eps, rowmask);
  return 0;
}
int row_nonzero_mask(Ctx& ctx, const SeqDev& s, const float* x, int ld, int C, float* mask) {
  LAUNCH_ROWS(k_row_nonzero, s, x, ld, C, mask);
  return 0;
}
int col0_nonzero_mask(Ctx& ctx, const SeqDev& s, const float* x, int ld, float* mask) {
  LAUNCH_ROWS(k_col0_nonzero, s, x, ld, mask);
  return 0;
}
int token_nonzero_mask(Ctx& ctx, const SeqDev& s, const int32_t* tok, float* mask) {
  LAUNCH_ROWS(k_tok_nonzero, s, tok, mask);
  return 0;
}
int positions_from_mask(Ctx& ctx, const SeqDev& s, const float* mask, int32_t* pos) {
  if (!ctx.dry && s.B > 0) {
    k_positions<<<s.B, 32, 0, ctx.stream>>>(s.utt, s.B, mask, pos);
    ++g_launches;
    SSB_CUDA(cudaGetLastError());
  }
  return 0;
}
int add_positional(Ctx& ctx, const SeqDev& s, float* x, int ld, int C, const int32_t* pos, const float* table,
                   int table_rows, const float* alpha_ptr) {
  LAUNCH_ROWS(k_add_positional, s, x, ld, C, pos, table, table_rows, alpha_ptr);
  return 0;
}
int embed_rows(Ctx& ctx, const SeqDev& s, const int32_t* idx, const float* table, int nt, float scale, float* x, int ld,
               int C, int accumulate) {
  LAUNCH_ROWS(k_embed, s, idx, table, nt, scale, x, ld, C, accumulate);
  return 0;
}
int note_encoder(Ctx& ctx, const SeqDev& s, const int32_t* note, const int32_t* type, const float* dur, const float* En,
                 const float* Et, const float* w, const float* b, float scale, float* x, int ld, int C, int accumulate) {
  LAUNCH_ROWS(k_note_encoder, s, note, type, dur, En, Et, w, b, scale, x, ld, C, accumulate);
  return 0;
}
int expand_states(Ctx& ctx, const SeqDev& fr, const SeqDev& ph, const int32_t* mel2ph, const float* src, int ld_s,
                  float* out, int ld_o, int C, const int32_t* note, int32_t* midi, float* tgt_nonpad) {
  LAUNCH_ROWS(k_expand, fr, ph.utt, mel2ph, src, ld_s, out, ld_o, C, note, midi, tgt_nonpad);
  return 0;
}
int combine_rows(Ctx& ctx, const SeqDev& s, const CombineArgs& a) {
  LAUNCH_ROWS(k_combine, s, a);
  return 0;
}
int scale_mask_add_rowscalar(Ctx& ctx, const SeqDev& s, const float* x, int ldx, int C, const float* mask,
                             const float* rowscalar, float* y, int ldy) {
  LAUNCH_ROWS(k_smar, s, x, ldx, C, mask, rowscalar, y, ldy);
  return 0;
}
int concat2_pos(Ctx& ctx, const SeqDev& s, const float* z, int C, const int32_t* pos, const float* table, int table_rows,
                float* out, int ldo) {
  LAUNCH_ROWS(k_concat2_pos, s, z, C, pos, table, table_rows, out, ldo);
  return 0;
}
int concat_cond(Ctx& ctx, const SeqDev& s, const float* coarse, const float* dec, const float* spk, const float* emo,
                const float* style, float* out, int ldo) {
  SSB_CHECK(ldo == 80 + 256 * (1 + (dec != nullptr) + (emo != nullptr) + (style != nullptr)),
            "concat_cond: ldo does not match the segments present");
  LAUNCH_ROWS(k_concat_cond, s, coarse, dec, spk, emo, style, out, ldo);
  return 0;
}
int clip_rows(Ctx& ctx, const SeqDev& s, float* x, int ld, int C, float lo, float hi) {
  LAUNCH_ROWS(k_clip, s, x, ld, C, lo, hi);
  return 0;
}
int dur_from_logits(Ctx& ctx, const SeqDev& s, const float* logdur, const float* nonpad, int32_t* dur) {
  LAUNCH_ROWS(k_dur, s, logdur, nonpad, dur);
  return 0;
}
int length_regulate(Ctx& ctx, const SeqDev& fr, const SeqDev& ph, const int32_t* dur, int32_t* mel2ph) {
  if (!ctx.dry && fr.B > 0) {
    k_length_regulate<<<fr.B, 256, (size_t)ph.maxlen * sizeof(int), ctx.stream>>>(fr.utt, ph.utt, dur, mel2ph);
    ++g_launches;
    SSB_CUDA(cudaGetLastError());
  }
  return 0;
}
int codebook_norms(Ctx& ctx, const float* cb, int n, float* out) {
  if (!ctx.dry) {
    k_cb_norm<<<(n + 7) / 8, dim3(32, 8), 0, ctx.stream>>>(cb, n, out);
    SSB_CUDA(cudaGetLastError());
  }
  return 0;
}
int rvq_lookup(Ctx& ctx, const SeqDev& s, const float* x, int ldx, const float* cb, const float* cbn, int n_embed,
               int depth, float* quant, int ldq, int32_t* codes) {
  LAUNCH_ROWS(k_rvq, s, x, ldx, cb, cbn, n_embed, depth, quant, ldq, codes);
  return 0;
}
int mel_q_sample(Ctx& ctx, const SeqDev& s, const float* coarse, int ldc, const float* noise, const float* smin,
                 const float* smax, float sa, float s1a, float* x, int ldx, const UttRng* rng, uint64_t sid) {
  LAUNCH_ROWS(k_mel_q_sample, s, rng, coarse, ldc, noise, smin, smax, sa, s1a, x, ldx, sid);
  return 0;
}
int mel_p_sample(Ctx& ctx, const SeqDev& s, float* x, int ldx, const float* eps, int lde, const float* noise,
                 const float* tab, const UttRng* rng, uint64_t sid, bool clip) {
  LAUNCH_ROWS(k_mel_p_sample, s, rng, x, ldx, eps, lde, noise, tab, sid, clip ? 1 : 0);
  return 0;
}
int plms_update(Ctx& ctx, const SeqDev& s, const PlmsArgs& a) {
  LAUNCH_ROWS(k_plms_update, s, a);
  return 0;
}
int mel_denorm(Ctx& ctx, const SeqDev& s, const float* x, int ldx, const float* smin, const float* smax,
               const float* rowmask, float* mel, int ld) {
  LAUNCH_ROWS(k_mel_denorm, s, x, ldx, smin, smax, rowmask, mel, ld);
  return 0;
}
int f0_p_sample(Ctx& ctx, const SeqDev& s, const F0StepArgs& a) {
  LAUNCH_ROWS(k_f0_p_sample, s, a);
  return 0;
}
int f0_init(Ctx& ctx, const SeqDev& s, float* z, int32_t* uv, const float* gnoise, const UttRng* rng, uint64_t sid) {
  LAUNCH_ROWS(k_f0_init, s, rng, z, uv, gnoise, sid);
  return 0;
}
int ddiff_input(Ctx& ctx, const SeqDev& s, const float* z, const int32_t* uv, const float* w, const float* b,
                const float* Euv, const float* d0, float* x, float* y, int C, __half* yh, __half* yl) {
  LAUNCH_ROWS(k_ddiff_input, s, z, uv, w, b, Euv, d0, x, y, C, yh, yl);
  return 0;
}
int midi_clip_band(Ctx& ctx, const SeqDev& s, const int32_t* midi, float* lo, float* hi) {
  LAUNCH_ROWS(k_midi_band, s, midi, lo, hi);
  return 0;
}
int pitch_glue(Ctx& ctx, const SeqDev& s, const PitchGlueArgs& a) {
  LAUNCH_ROWS(k_pitch_glue, s, a);
  return 0;
}
int pitch_glue_conv(Ctx& ctx, const SeqDev& s, const PitchGlueConvArgs& a) {
  LAUNCH_ROWS(k_pitch_glue_conv, s, a);
  return 0;
}

size_t nsf_scratch_doubles(const SeqDev& s256) { return (size_t)(s256.total * 9 * sizeof(float) + 7) / 8 + 8; }

int nsf_source(Ctx& ctx, const SeqDev& s1, const SeqDev& s256, const float* f0, const float* lw, const float* lb,
               const float* rand_ini, const float* noise, float* har, double* scratch, int upp, float sr) {
  if (ctx.dry || s1.B == 0) return 0;
  float* sines = reinterpret_cast<float*>(scratch);
  k_nsf_phase<<<dim3(9, s1.B), 256, 0, ctx.stream>>>(s1.utt, s256.utt, s1.rng, f0, rand_ini, sines, upp, sr);
  SSB_CUDA(cudaGetLastError());
  k_nsf_merge<<<dim3((s256.maxlen + 255) / 256, s1.B), 256, 0, ctx.stream>>>(s1.utt, s256.utt, s256.rng, f0, sines, noise,
                                                                            lw, lb, har, upp);
  SSB_CUDA(cudaGetLastError());
  g_launches += 2;
  return 0;
}
int noise_conv_add(Ctx& ctx, const SeqDev& sx, const SeqDev& s256, float* x, int ld, int C, const float* har,
                   const float* w, const float* b, int s, __half* ph, __half* pl, float pslope, const float* wt) {
  if (ctx.dry || sx.B == 0) return 0;
  if (wt && C % 4 == 0 && ld % 4 == 0) {
    const int K = s == 1 ? 1 : 2 * s;
    const size_t smem = ((size_t)NC_TR * s + K) * sizeof(float);
    k_noise_conv_add_tiled<<<dim3((sx.maxlen + NC_TR - 1) / NC_TR, sx.B), 256, smem, ctx.stream>>>(sx.utt, s256.utt, x, ld, C, har, wt, b, s,
                                                                                             ph, pl, pslope);
  } else {
    k_noise_conv_add<<<row_grid(sx), dim3(32, RPB), 0, ctx.stream>>>(sx.utt, s256.utt, x, ld, C, har, w, b, s, ph, pl, pslope);
  }
    ++g_launches;
  SSB_CUDA(cudaGetLastError());
  return 0;
}
int tanh_out(Ctx& ctx, const SeqDev& s, const float* x, int ld, float* wav) {
  if (ctx.dry || s.B == 0) return 0;
  k_tanh_out<<<dim3((s.maxlen + 255) / 256, s.B), 256, 0, ctx.stream>>>(s.utt, x, ld, wav);
    ++g_launches;
  SSB_CUDA(cudaGetLastError());
  return 0;
}
int conv_post_tanh(Ctx& ctx, const SeqDev& s, const float* x, int ld, int C, int taps, int center, const float* W, int npad,
                   const float* bias, float slope, float* wav) {
  if (ctx.dry || s.B == 0) return 0;
  SSB_CHECK(C % 4 == 0 && ld % 4 == 0, "conv_post_tanh: channel count must be a multiple of 4");
  const size_t smem = ((size_t)(CP_T + taps - 1) * (C + 1) + (size_t)taps * C) * sizeof(float);
  SSB_CHECK(smem <= 48 * 1024, "conv_post_tanh: window does not fit the default shared-memory limit");
  k_conv_post_tanh<<<dim3((s.maxlen + CP_T - 1) / CP_T, s.B), CP_T, smem, ctx.stream>>>(s.utt, x, ld, C, taps, center, W, npad, bias, slope, wav);
  ++g_launches;
  SSB_CUDA(cudaGetLastError());
  return 0;
}
int mel_postprocess(Ctx& ctx, const SeqDev& s, float* mel, int ld, float* f0, float vmin, float vmax) {
  LAUNCH_ROWS(k_mel_post, s, mel, ld, f0, vmin, vmax);
  return 0;
}

}  // namespace ssb
