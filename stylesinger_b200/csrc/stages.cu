// Stage drivers: compose the kernels into the reference's modules (one function per SURVEY.md §8a group).
#include <string.h>

#include "philox.cuh"
#include "sampler_tc.cuh"
#include "stages.cuh"

namespace ssb {

ConvGemm make_gemm(const Conv& c, const SeqDev& s, const float* A, int lda) {
  ConvGemm g;
  g.A = A; g.lda = lda; g.Cin = c.Cin; g.taps = c.taps; g.dil = c.dil; g.center = c.center;
  g.W = c.W; g.N = c.N; g.Npad = c.Npad; g.tiles = s.tiles; g.ntiles = s.ntiles;
  g.e.bias = c.bias;
  return g;
}
GemmTC make_gemm_tc(const ConvTC& w, const SeqDev& s, const __half* A_hi, const __half* A_lo) {
  GemmTC g;
  g.A_hi = A_hi; g.A_lo = A_lo; g.rows_total = s.rows; g.w = &w; g.tiles = s.tiles; g.ntiles = s.ntiles;
  g.e.mode = EPI_GENERIC;
  return g;
}

int run_dense(Ctx& c, const Dense& d, bool tc, const SeqDev& s, const DenseIn& in, const Epi& e, bool single_pass) {
  SSB_CHECK(!e.bias, "run_dense: the bias is the layer's own");
  if (!tc) {
    SSB_CHECK(in.x != nullptr, "run_dense: the fp32 kernel needs the input as fp32 rows");
    ConvGemm g = make_gemm(d.f, s, in.x, in.ld);
    g.a_act = in.act; g.a_slope = in.slope;
    g.e = e;
    g.e.bias = d.f.bias;
    return conv_gemm(c, g);
  }
  SSB_CHECK(d.t.ok && in.hi && in.lo, "run_dense: the tensor-core kernel needs eligible weights and the input as fp16 planes");
  SSB_CHECK(e.mode == EPI_GENERIC && !e.add && e.beta == 1.0f && !e.out2,
            "run_dense: the tensor-core kernel's generic epilogue has no gate / skip mode, addend, beta or second fp32 output");
  GemmTC g = make_gemm_tc(d.t, s, in.hi, in.lo);
  g.single_pass = single_pass;
  EpiTC& t = g.e;
  t.out = e.out; t.ldo = e.ldo;
  t.oh = e.out2_h; t.ol = e.out2_l; t.ldh = e.ldh; t.vec2 = e.vec2;
  t.plane_act = e.plane_act; t.plane_slope = e.plane_slope;
  t.res = e.res; t.ld_res = e.ld_res; t.rowmask = e.rowmask;
  t.alpha = e.alpha; t.act = e.act; t.act_slope = e.act_slope;
  t.accum = e.accum; t.gamma = e.gamma;
  return conv_gemm_tc(c, g);
}

bool long_batch_tc(const Model& m, const SeqDev& s) { return m.use_tc && m.fft_tc && tc_available() && s.ntiles >= 8; }

int upload_layout(Ctx& c, const Seq& s, int rate, SeqDev* out) {
  const int nt = s.ntiles(rate);
  int2* tiles = c.alloc<int2>((size_t)nt + 1);
  int4* utt = c.alloc<int4>((size_t)s.B + 1);
  UttRng* rng = c.alloc<UttRng>((size_t)s.B + 1);
  int4* tpos = c.alloc<int4>((size_t)nt + 1);
  out->tile_pos = tpos;
  out->tiles = tiles; out->ntiles = nt; out->utt = utt; out->rng = rng; out->B = s.B; out->rows = s.rows(rate);
  out->total = s.total * rate; out->maxlen = s.maxlen * rate; out->rate = rate;
  if (c.dry) return 0;
  SSB_CHECK(!c.failed && tiles && utt && rng && tpos, "workspace too small (layout tables)");
  std::vector<int2> ht((size_t)nt + 1);
  std::vector<int4> hu((size_t)s.B + 1);
  std::vector<UttRng> hr((size_t)s.B + 1);
  std::vector<int4> htp((size_t)nt + 1);
  int k = 0;
  int64_t tight = 0;
  for (int b = 0; b < s.B; ++b) {
    const int len = s.len[b] * rate;
    const int rs = s.rs[b] * rate;
    hu[b] = make_int4(rs, len, (int)tight, 0);
    hr[b] = s.utt_seeds ? UttRng{s.utt_seeds[b], 0, 0} : UttRng{s.seed, (int32_t)tight, b};
    for (int t0 = 0; t0 < len; t0 += TILE_M) {
      htp[k] = make_int4((int)tight + t0, b, t0, 0);
      ht[k++] = make_int2(rs + t0, (len - t0) < TILE_M ? (len - t0) : TILE_M);
    }
    tight += len;
  }
  SSB_CUDA(cudaMemcpyAsync(tpos, htp.data(), sizeof(int4) * nt, cudaMemcpyHostToDevice, c.stream));
  SSB_CUDA(cudaMemcpyAsync(tiles, ht.data(), sizeof(int2) * nt, cudaMemcpyHostToDevice, c.stream));
  SSB_CUDA(cudaMemcpyAsync(utt, hu.data(), sizeof(int4) * s.B, cudaMemcpyHostToDevice, c.stream));
  SSB_CUDA(cudaMemcpyAsync(rng, hr.data(), sizeof(UttRng) * s.B, cudaMemcpyHostToDevice, c.stream));
  // pageable-source async copies are staged before returning, so the host vectors may die here
  return 0;
}

float* alloc_rows(Ctx& c, const SeqDev& s, int C, bool zero) {
  float* p = c.alloc<float>((size_t)s.rows * C);
  if (!c.dry && p && !c.failed && zero) cudaMemsetAsync(p, 0, (size_t)s.rows * C * sizeof(float), c.stream);
  return p;
}
int32_t* alloc_rows_i32(Ctx& c, const SeqDev& s, int C) {
  int32_t* p = c.alloc<int32_t>((size_t)s.rows * C);
  if (!c.dry && p && !c.failed) cudaMemsetAsync(p, 0, (size_t)s.rows * C * sizeof(int32_t), c.stream);
  return p;
}
__half* alloc_half_rows(Ctx& c, const SeqDev& s, int C) {
  __half* p = c.alloc<__half>((size_t)s.rows * C);
  if (!c.dry && p && !c.failed) cudaMemsetAsync(p, 0, (size_t)s.rows * C * sizeof(__half), c.stream);
  return p;
}

// ------------------------------------------------------------------------------------------------
// a2-a5: FFTBlocks body (tts_modules.py:293-305 + EncSALayer common_layers.py:649-673)
// x [rows,256] in/out; keep = 1 - padding_mask (row mask, also the key mask)
int fft_blocks(Ctx& c, const FFT& f, const SeqDev& s, float* x, const float* keep, bool tc) {
  const int H = 256;
  const size_t mk = c.mark();
  tc = tc && f.tc_ok;
  float* h = alloc_rows(c, s, H);
  float* qkv = alloc_rows(c, s, 3 * H);
  float* att = alloc_rows(c, s, H);
  float* ff = tc ? nullptr : alloc_rows(c, s, 4 * H);
  __half *hh = nullptr, *hl = nullptr, *fh = nullptr, *fl = nullptr;  // fp16 hi/lo planes of h and of gelu(ffn_1)
  // wgmma attention (attention_tc.cu): q/k/v only as fp16 hi/lo planes [rows, 768] + V^T planes [256, ldvt]
  const bool atc = tc && attention_tc_enabled();
  const int64_t ldvt = (s.rows + 7) & ~int64_t(7);
  __half *qh = nullptr, *ql = nullptr, *vth = nullptr, *vtl = nullptr;
  if (tc) {
    hh = alloc_half_rows(c, s, H); hl = alloc_half_rows(c, s, H);
    fh = alloc_half_rows(c, s, 4 * H); fl = alloc_half_rows(c, s, 4 * H);
  }
  if (atc) {
    qh = alloc_half_rows(c, s, 3 * H); ql = alloc_half_rows(c, s, 3 * H);
    vth = c.alloc<__half>((size_t)ldvt * H); vtl = c.alloc<__half>((size_t)ldvt * H);
  }
  WS_OK(c);
  for (size_t i = 0; i < f.layers.size(); ++i) {
    const FFTLayer& L = f.layers[i];
    RUN(layernorm_rows(c, s, x, H, h, H, H, L.ln1_g, L.ln1_b, 1e-5f, nullptr));
    if (tc) RUN(split_planes(c, h, H, s.rows, H, 1.0f, hh, hl));
    {
      Epi e;
      if (atc) { e.out2_h = qh; e.out2_l = ql; e.ldh = 3 * H; }
      else { e.out = qkv; e.ldo = 3 * H; }
      RUN(run_dense(c, L.qkv, tc, s, {h, H, hh, hl}, e));
    }
    if (atc) {
      RUN(transpose_planes(c, qh, ql, 3 * H, 2 * H, s.rows, H, vth, vtl, ldvt));
      AttnTCArgs a;
      a.utt_q = s.utt; a.utt_k = s.utt; a.B = s.B; a.max_q = s.maxlen; a.heads = 2;
      a.Qh = qh; a.Ql = ql; a.rows_q = s.rows; a.ldq = 3 * H; a.qcol0 = 0;
      a.Kh = qh; a.Kl = ql; a.rows_k = s.rows; a.ldk = 3 * H; a.kcol0 = H;
      a.Vth = vth; a.Vtl = vtl; a.ldvt = ldvt;
      a.keymask = keep; a.scale = 0.08838834764831845f;  // 128^-0.5
      a.oh = hh; a.ol = hl; a.ldh = H;                   // straight into the out-projection's A planes
      RUN(attention_tc(c, a));
    } else {
      AttnArgs a;
      a.utt_q = s.utt; a.utt_k = s.utt; a.B = s.B; a.max_q = s.maxlen; a.heads = 2;
      a.Q = qkv; a.ldq = 3 * H; a.K = qkv + H; a.ldk = 3 * H; a.V = qkv + 2 * H; a.ldv = 3 * H;
      a.keymask = keep; a.scale = 0.08838834764831845f;  // 128^-0.5
      a.out = att; a.ldo = H;
      RUN(attention(c, a));
    }
    if (tc && !atc) RUN(split_planes(c, att, H, s.rows, H, 1.0f, hh, hl));
    Epi eres;  // x = (x + layer output) * keep: the epilogue of the out-projection and of ffn_2
    eres.res = x; eres.ld_res = H; eres.rowmask = keep; eres.out = x; eres.ldo = H;
    RUN(run_dense(c, L.out, tc, s, {att, H, hh, hl}, eres));
    RUN(layernorm_rows(c, s, x, H, h, H, H, L.ln2_g, L.ln2_b, 1e-5f, nullptr));
    if (tc) RUN(split_planes(c, h, H, s.rows, H, 1.0f, hh, hl));
    {  // TransformerFFNLayer (transformer.py): ffn_2(gelu(ffn_1(x) * k^-0.5)); on tensor cores gelu(ffn_1) exists only as planes
      Epi e;
      e.alpha = 1.0f / sqrtf((float)f.kernel); e.act = ACT_GELU;
      if (tc) { e.out2_h = fh; e.out2_l = fl; e.ldh = 4 * H; }
      else { e.out = ff; e.ldo = 4 * H; }
      RUN(run_dense(c, L.ffn1, tc, s, {h, H, hh, hl}, e));
    }
    RUN(run_dense(c, L.ffn2, tc, s, {ff, 4 * H, fh, fl}, eres));
  }
  // final LN * mask, in place via h
  RUN(layernorm_rows(c, s, x, H, h, H, H, f.ln_g, f.ln_b, 1e-5f, keep));
  if (!c.dry) SSB_CUDA(cudaMemcpyAsync(x, h, (size_t)s.rows * H * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  c.release(mk);
  return 0;
}

// a1 + a7: encoder_out = FastspeechEncoder(txt) + NoteEncoder(note, dur, type)
int run_encoder(Ctx& c, const Model& m, const SeqDev& sp, const int32_t* tok_g, const int32_t* note_g,
                const int32_t* type_g, const float* ndur_g, float* srcmask, float* enc_out) {
  const int H = 256;
  const size_t mk = c.mark();
  int32_t* pos = alloc_rows_i32(c, sp);
  WS_OK(c);
  RUN(token_nonzero_mask(c, sp, tok_g, srcmask));
  RUN(positions_from_mask(c, sp, srcmask, pos));
  RUN(embed_rows(c, sp, tok_g, m.tok_emb, m.n_tokens, 16.0f, enc_out, H, H, 0));
  RUN(add_positional(c, sp, enc_out, H, H, pos, m.pos_table, m.pos_rows, nullptr));
  // FFTBlocks.forward: x = x.transpose * nonpadding (tts_modules.py:293)
  {
    CombineArgs a;
    a.m[0] = enc_out; a.ldm[0] = H; a.rowmask = srcmask; a.out = enc_out; a.ldo = H; a.C = H;
    RUN(combine_rows(c, sp, a));
  }
  RUN(fft_blocks(c, m.enc, sp, enc_out, srcmask));
  // StyleSinger.forward: encoder_out + note_encoder(note, note_dur, note_type) (stylesinger.py:124-126); a null note_g
  // stops at FastspeechEncoder.forward (the FS_ENCODERS['fft'] drop-in, ssb_fft_encoder)
  if (note_g) RUN(note_encoder(c, sp, note_g, type_g, ndur_g, m.note_emb, m.type_emb, m.dur_w, m.dur_b, 16.0f, enc_out, H, H, 1));
  c.release(mk);
  return 0;
}

// a16 body: FastspeechDecoder.forward = FFTBlocks.forward(x) with the padding mask taken from x itself
// (tts_modules.py:281-306): xd [rows,256] in/out
int run_fft_decoder(Ctx& c, const Model& m, const SeqDev& sf, const float* dec_in, float* xd, bool tc) {
  const int H = 256;
  const size_t mk = c.mark();
  float* keep = alloc_rows(c, sf, 1);
  float* c0 = alloc_rows(c, sf, 1);
  int32_t* pos = alloc_rows_i32(c, sf);
  WS_OK(c);
  if (!c.dry && xd != dec_in)
    SSB_CUDA(cudaMemcpyAsync(xd, dec_in, (size_t)sf.rows * H * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  RUN(row_nonzero_mask(c, sf, dec_in, H, H, keep));
  RUN(col0_nonzero_mask(c, sf, dec_in, H, c0));
  RUN(positions_from_mask(c, sf, c0, pos));
  RUN(add_positional(c, sf, xd, H, H, pos, m.pos_table, m.pos_rows, m.dec.pos_alpha));
  {
    CombineArgs a;
    a.m[0] = xd; a.ldm[0] = H; a.rowmask = keep; a.out = xd; a.ldo = H; a.C = H;
    RUN(combine_rows(c, sf, a));
  }
  RUN(fft_blocks(c, m.dec, sf, xd, keep, tc));
  c.release(mk);
  return 0;
}

// a8: DurationPredictor.inference (tts_modules.py:105-130)
int run_duration_predictor(Ctx& c, const Model& m, const SeqDev& sp, const float* dur_inp, const float* srcmask,
                           float* logdur /*[rows]*/, int32_t* dur /*[rows]*/) {
  const int H = 256;
  const size_t mk = c.mark();
  float* a = alloc_rows(c, sp, H);
  float* b = alloc_rows(c, sp, H);
  WS_OK(c);
  const float* cur = dur_inp;
  for (int i = 0; i < m.dp_layers; ++i) {
    ConvGemm g = make_gemm(m.dp_conv[i], sp, cur, H);
    g.e.act = ACT_RELU; g.e.out = a; g.e.ldo = H;
    RUN(conv_gemm(c, g));
    RUN(layernorm_rows(c, sp, a, H, b, H, H, m.dp_ln_g[i], m.dp_ln_b[i], 1e-5f, srcmask));
    cur = b;  // next conv reads b and writes a; the LN after it overwrites b only once that conv has finished
  }
  {
    ConvGemm g = make_gemm(m.dp_lin, sp, cur, H);
    g.e.rowmask = srcmask; g.e.out = logdur; g.e.ldo = 1;
    RUN(conv_gemm(c, g));
  }
  RUN(dur_from_logits(c, sp, logdur, srcmask, dur));
  c.release(mk);
  return 0;
}

// f0_gen 'conv': PitchPredictor.forward (tts_modules.py:221-234), eval mode.  x [rows,256] -> out [rows,2].  No mask
// anywhere, as in the reference: every buffer's guard rows stay zero, which is the SAME padding of a B=1 call.
int run_pitch_predictor(Ctx& c, const Model& m, int which, const SeqDev& s, const float* x_g, float* out_g, bool tc) {
  const int H = 256;
  SSB_CHECK(m.f0_gen == SSB_F0_GEN_CONV, "pitch predictor: the model was not created with SSB_F0_GEN_CONV");
  SSB_CHECK(which == 0 || which == 1, "pitch predictor: which must be 0 (pitch_predictor) or 1 (pitch_inpainter_predictor)");
  const PitchPredictor& p = m.pp[which];
  tc = tc && p.tc_ok;
  const size_t mk = c.mark();
  float* xs = alloc_rows(c, s, H);
  float* a = alloc_rows(c, s, H);
  float* b = alloc_rows(c, s, H);
  float* c0 = alloc_rows(c, s, 1);
  int32_t* pos = alloc_rows_i32(c, s);
  __half *hh = nullptr, *hl = nullptr;
  if (tc) {
    hh = alloc_half_rows(c, s, H);
    hl = alloc_half_rows(c, s, H);
  }
  WS_OK(c);
  // positions = pos_embed_alpha * embed_positions(xs[..., 0]); xs = xs + positions
  if (!c.dry) SSB_CUDA(cudaMemcpyAsync(xs, x_g, (size_t)s.rows * H * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  RUN(col0_nonzero_mask(c, s, xs, H, c0));
  RUN(positions_from_mask(c, s, c0, pos));
  RUN(add_positional(c, s, xs, H, H, pos, m.pos_table, m.pos_rows, p.pos_alpha));
  const float* cur = xs;
  for (int i = 0; i < PitchPredictor::kLayers; ++i) {
    // ConstantPad1d + Conv1d + ReLU (the guard rows are the zero pad), then LayerNorm(dim=1); Dropout is off
    if (tc) RUN(split_planes(c, cur, H, s.rows, H, 1.0f, hh, hl));
    Epi e;
    e.act = ACT_RELU; e.out = a; e.ldo = H;
    RUN(run_dense(c, p.conv[i], tc, s, {cur, H, hh, hl}, e));
    RUN(layernorm_rows(c, s, a, H, b, H, H, p.ln_g[i], p.ln_b[i], 1e-5f, nullptr));
    cur = b;  // the next conv reads b and writes a; the LN after it overwrites b only once that conv has finished
  }
  {
    ConvGemm g = make_gemm(p.linear, s, cur, H);
    g.e.out = out_g; g.e.ldo = 2;
    RUN(conv_gemm(c, g));
  }
  c.release(mk);
  return 0;
}

// a10-a12: get_style (stylesinger.py:189-214)
int run_style(Ctx& c, const Model& m, const SeqDev& sf, const SeqDev& sr, const float* dec0, const float* ref_g /*[rows,80]*/,
              const float* reff0_g /*[rows]*/, float* style /*[rows_f,256]*/, int32_t* codes /*[rows_r,depth] guarded*/,
              float* rq_in_out /*optional guarded [rows_r,256]*/) {
  const int H = 256;
  const size_t mk = c.mark();
  float* rmask = alloc_rows(c, sr, 1);
  float* x = alloc_rows(c, sr, 80);
  float* z = alloc_rows(c, sr, 80);
  float* wout = alloc_rows(c, sr, 80);
  float* h80 = alloc_rows(c, sr, 80);
  float* g160 = alloc_rows(c, sr, 160);
  float* np0 = alloc_rows(c, sr, 1);
  float* npi = alloc_rows(c, sr, 1);
  float* st = alloc_rows(c, sr, H);
  float* zq = alloc_rows(c, sr, H);
  float* cat = alloc_rows(c, sr, 2 * H);
  float* zl = alloc_rows(c, sr, H);
  float* kmask = alloc_rows(c, sr, 1);
  int32_t* pos = alloc_rows_i32(c, sr);
  float* kv = alloc_rows(c, sr, 2 * H);
  float* q = alloc_rows(c, sf, H);
  float* att = alloc_rows(c, sf, H);
  float* tmp = alloc_rows(c, sf, H);
  // long batches: the aligner's five projections per layer on the tensor-core kernel (the 256 -> 2048 -> 256 feed-forward is
  // 90 % of its FLOPs; its hidden activation then only exists as fp16 hi/lo planes); attention itself stays fp32
  const bool tc = long_batch_tc(m, sf) && m.align_tc_ok;
  float* hid = tc ? nullptr : alloc_rows(c, sf, 2048);
  WS_OK(c);
  // LocalStyleAdaptor.forward (lse.py:103-129)
  RUN(col0_nonzero_mask(c, sr, ref_g, 80, rmask));
  if (!c.dry) SSB_CUDA(cudaMemcpyAsync(x, ref_g, (size_t)sr.rows * 80 * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  for (int i = 0; i < 4; ++i) {  // WN.forward (wavenet.py:54-78), g=None
    {
      ConvGemm g = make_gemm(m.wn_in[i], sr, x, 80);
      g.e.mode = EPI_GATE; g.e.out = z; g.e.ldo = 80;
      RUN(conv_gemm(c, g));
    }
    ConvGemm g = make_gemm(m.wn_rs[i], sr, z, 80);
    if (i < 3) {
      g.e.mode = EPI_RES_SKIP; g.e.C = 80; g.e.res = x; g.e.ld_res = 80; g.e.beta = 1.0f; g.e.rowmask = rmask;
      g.e.out = x; g.e.ldo = 80; g.e.skip = wout; g.e.ld_skip = 80; g.e.skip_init = (i == 0);
    } else {
      g.e.out = wout; g.e.ldo = 80; g.e.accum = 1; g.e.gamma = 1.0f;
    }
    RUN(conv_gemm(c, g));
  }
  // ref_ph = wn_out * mask + ref_f0 broadcast (lse.py:110,121-123)
  RUN(scale_mask_add_rowscalar(c, sr, wout, 80, 80, rmask, reff0_g, x, 80));
  // ConvBlocks (lse.py:229-240)
  RUN(row_nonzero_mask(c, sr, x, 80, 80, np0));
  for (int i = 0; i < 5; ++i) {
    RUN(row_nonzero_mask(c, sr, x, 80, 80, npi));
    for (int j = 0; j < 2; ++j) {
      const Model::CB& b = m.cb[i * 2 + j];
      RUN(layernorm_rows(c, sr, x, 80, h80, 80, 80, b.ln_g, b.ln_b, 1e-5f, nullptr));
      {
        ConvGemm g = make_gemm(b.c1, sr, h80, 80);
        g.e.alpha = 1.0f / sqrtf(5.0f); g.e.act = ACT_GELU; g.e.out = g160; g.e.ldo = 160;
        RUN(conv_gemm(c, g));
      }
      {
        ConvGemm g = make_gemm(b.c2, sr, g160, 160);
        g.e.res = x; g.e.ld_res = 80; g.e.rowmask = npi; g.e.out = x; g.e.ldo = 80;
        RUN(conv_gemm(c, g));
      }
    }
  }
  {
    CombineArgs a;
    a.m[0] = x; a.ldm[0] = 80; a.rowmask = np0; a.out = x; a.ldo = 80; a.C = 80;
    RUN(combine_rows(c, sr, a));
  }
  RUN(layernorm_rows(c, sr, x, 80, h80, 80, 80, m.cb_last_g, m.cb_last_b, 1e-5f, np0));
  {
    ConvGemm g = make_gemm(m.cb_post, sr, h80, 80);
    g.e.rowmask = np0; g.e.out = st; g.e.ldo = H;
    RUN(conv_gemm(c, g));
  }
  if (rq_in_out && !c.dry)
    SSB_CUDA(cudaMemcpyAsync(rq_in_out, st, (size_t)sr.rows * H * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  RUN(rvq_lookup(c, sr, st, H, m.codebooks, m.cb_norm2, m.hp.n_rq, m.hp.rq_depth, zq, H, codes));
  // positions + l1 (stylesinger.py:198-200)
  RUN(col0_nonzero_mask(c, sr, zq, H, kmask));
  RUN(positions_from_mask(c, sr, kmask, pos));
  RUN(concat2_pos(c, sr, zq, H, pos, m.pos_table, m.pos_rows, cat, 2 * H));
  {
    ConvGemm g = make_gemm(m.l1, sr, cat, 2 * H);
    g.e.out = zl; g.e.ldo = H;
    RUN(conv_gemm(c, g));
  }
  RUN(col0_nonzero_mask(c, sr, zl, H, kmask));  // style_key_padding_mask = zl[:,:,0].eq(0) (:204) -> attend where != 0
  // ProsodyAligner (lse.py:59-81), forcing=False
  if (!c.dry) SSB_CUDA(cudaMemcpyAsync(style, dec0, (size_t)sf.rows * H * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  __half *sth = nullptr, *stl = nullptr, *zlh = nullptr, *zll = nullptr, *hdh = nullptr, *hdl = nullptr;
  if (tc) {
    sth = alloc_half_rows(c, sf, H); stl = alloc_half_rows(c, sf, H);
    zlh = alloc_half_rows(c, sr, H); zll = alloc_half_rows(c, sr, H);
    hdh = alloc_half_rows(c, sf, 2048); hdl = alloc_half_rows(c, sf, 2048);
    WS_OK(c);
    RUN(split_planes(c, zl, H, sr.rows, H, 1.0f, zlh, zll));
  }
  const bool atc = tc && attention_tc_enabled();
  const int64_t ldvt = (sr.rows + 7) & ~int64_t(7);
  __half *aqh = nullptr, *aql = nullptr, *akh = nullptr, *akl = nullptr, *avth = nullptr, *avtl = nullptr;
  if (atc) {
    aqh = alloc_half_rows(c, sf, H); aql = alloc_half_rows(c, sf, H);
    akh = alloc_half_rows(c, sr, 2 * H); akl = alloc_half_rows(c, sr, 2 * H);
    avth = c.alloc<__half>((size_t)ldvt * H); avtl = c.alloc<__half>((size_t)ldvt * H);
    WS_OK(c);
  }
  for (int i = 0; i < 2; ++i) {
    const AlignLayer& L = m.align[i];
    if (tc) RUN(split_planes(c, style, H, sf.rows, H, 1.0f, sth, stl));
    {
      Epi e;
      if (atc) { e.out2_h = aqh; e.out2_l = aql; e.ldh = H; }
      else { e.out = q; e.ldo = H; }
      RUN(run_dense(c, L.q, tc, sf, {style, H, sth, stl}, e));
    }
    {
      Epi e;
      if (atc) { e.out2_h = akh; e.out2_l = akl; e.ldh = 2 * H; }
      else { e.out = kv; e.ldo = 2 * H; }
      RUN(run_dense(c, L.kv, tc, sr, {zl, H, zlh, zll}, e));
    }
    if (atc) {  // cross-attention on the tensor-core kernel: q planes [F rows, 256], k | v planes [R rows, 512]
      RUN(transpose_planes(c, akh, akl, 2 * H, H, sr.rows, H, avth, avtl, ldvt));
      AttnTCArgs a;
      a.utt_q = sf.utt; a.utt_k = sr.utt; a.B = sf.B; a.max_q = sf.maxlen; a.heads = 2;
      a.Qh = aqh; a.Ql = aql; a.rows_q = sf.rows; a.ldq = H; a.qcol0 = 0;
      a.Kh = akh; a.Kl = akl; a.rows_k = sr.rows; a.ldk = 2 * H; a.kcol0 = 0;
      a.Vth = avth; a.Vtl = avtl; a.ldvt = ldvt;
      a.keymask = kmask; a.scale = 0.08838834764831845f;
      a.oh = sth; a.ol = stl; a.ldh = H;
      RUN(attention_tc(c, a));
    } else {
      AttnArgs a;
      a.utt_q = sf.utt; a.utt_k = sr.utt; a.B = sf.B; a.max_q = sf.maxlen; a.heads = 2;
      a.Q = q; a.ldq = H; a.K = kv; a.ldk = 2 * H; a.V = kv + H; a.ldv = 2 * H;
      a.keymask = kmask; a.scale = 0.08838834764831845f; a.out = att; a.ldo = H;
      RUN(attention(c, a));
    }
    if (tc && !atc) RUN(split_planes(c, att, H, sf.rows, H, 1.0f, sth, stl));
    Epi eres;  // tmp = style + layer output: the epilogue of the out-projection and of linear2
    eres.res = style; eres.ld_res = H; eres.out = tmp; eres.ldo = H;
    RUN(run_dense(c, L.out, tc, sf, {att, H, sth, stl}, eres));
    RUN(layernorm_rows(c, sf, tmp, H, style, H, H, L.n1_g, L.n1_b, 1e-5f, nullptr));
    if (tc) RUN(split_planes(c, style, H, sf.rows, H, 1.0f, sth, stl));
    {
      Epi e;
      e.act = ACT_RELU;
      if (tc) { e.out2_h = hdh; e.out2_l = hdl; e.ldh = 2048; }
      else { e.out = hid; e.ldo = 2048; }
      RUN(run_dense(c, L.lin1, tc, sf, {style, H, sth, stl}, e));
    }
    RUN(run_dense(c, L.lin2, tc, sf, {hid, 2048, hdh, hdl}, eres));
    RUN(layernorm_rows(c, sf, tmp, H, style, H, H, L.n2_g, L.n2_b, 1e-5f, nullptr));
  }
  c.release(mk);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// a13/a18: the denoiser residual stack for one diffusion step.
// On entry b.x holds the residual stream and (b.y | b.yh,b.yl) holds x + d[t][0]; both are overwritten.
// SIMT path: fp32 conv_gemm.  Tensor-core path (b.tc): wgmma GEMMs on fp16 hi/lo planes.

// skip_projection + output_projection of the denoiser (net.py:126-130 / :262-266)
static int denoiser_heads(Ctx& c, const Denoiser& d, const SeqDev& s, DenoiserBufs& b) {
  const int C = d.C, L = d.L;
  if (b.tc_heads) {
    {  // skip_projection (1/sqrt(L) folded into the packed weights) + ReLU -> planes
      GemmTC g = make_gemm_tc(d.skip_tc, s, b.skh, b.skl);
      g.single_pass = b.single_pass;
      g.e.bias = d.skip_bias_pad; g.e.act = ACT_RELU; g.e.oh = b.sh; g.e.ol = b.sl; g.e.ldh = C;
      g.e.n_valid = C;
      RUN(conv_gemm_tc(c, g));
    }
    {  // output_projection (N padded to a tile multiple; only the first out_dims columns are meaningful)
      GemmTC g = make_gemm_tc(d.out_tc, s, b.sh, b.sl);
      g.single_pass = b.single_pass;
      g.e.bias = d.out_bias_pad; g.e.out = b.head; g.e.ldo = b.ld_head;
      g.e.n_valid = (d.out_dims + 31) / 32 * 32;
      RUN(conv_gemm_tc(c, g));
    }
    return 0;
  }
  {
    ConvGemm g = make_gemm(d.skip_proj, s, b.skip, C);
    g.a_scale = 1.0f / sqrtf((float)L);
    g.e.act = ACT_RELU; g.e.out = b.sbuf; g.e.ldo = C;
    RUN(conv_gemm(c, g));
  }
  {
    ConvGemm g = make_gemm(d.out_proj, s, b.sbuf, C);
    g.e.out = b.head; g.e.ldo = b.ld_head;
    RUN(conv_gemm(c, g));
  }
  return 0;
}

int denoiser_stack(Ctx& c, const Denoiser& d, const SeqDev& s, int t, DenoiserBufs& b) {
  const int C = d.C, L = d.L;
  SSB_CHECK(d.dtab != nullptr && t >= 0 && t < d.T, "denoiser: schedule not set (ssb_model_set_schedule) or bad t");
  const float* dt = d.dtab + (size_t)t * L * C;
  for (int l = 0; l < L; ++l) {  // residual layer l (net.py:66-78)
    if (b.tc) {
      {
        GemmTC g = make_gemm_tc(d.layers[l].dil.t, s, b.yh, b.yl);
        g.single_pass = b.single_pass;
        // K = 3*C (taps of y); the hoisted conditioner projection arrives as an epilogue addend (one [rows, 2C] matrix per layer)
        g.e.add = b.condpre + (size_t)l * (size_t)s.rows * 2 * C; g.e.ld_add = 2 * C;
        g.e.mode = EPI_GATE; g.e.bias = d.layers[l].bias_gate_tc;
        g.e.oh = b.zh; g.e.ol = b.zl; g.e.ldh = C;
        RUN(conv_gemm_tc(c, g));
      }
      GemmTC g = make_gemm_tc(d.layers[l].outp.t, s, b.zh, b.zl);
      g.single_pass = b.single_pass;
      // residual stream carried ONLY as the fp16 hi/lo planes of y = x + step bias (in place: this epilogue reads
      // y_l[row] and writes y_{l+1}[row] for the same rows/columns): no fp32 x is read or written in the T x L loop
      g.e.mode = EPI_RES_SKIP; g.e.C = C; g.e.beta = 0.70710678118654752440f;
      g.e.rh = b.yh; g.e.rl = b.yl; g.e.ld_rh = C; g.e.vec1 = dt + (size_t)l * C;
      if (l + 1 < L) { g.e.oh = b.yh; g.e.ol = b.yl; g.e.ldh = C; g.e.vec2 = dt + (size_t)(l + 1) * C; }
      g.e.skip = b.skip; g.e.ld_skip = C; g.e.skip_init = (l == 0);
      g.e.skip_tiled = b.tc_heads ? 1 : 0;
      if (b.tc_heads && l == L - 1) { g.e.sh = b.skh; g.e.sl = b.skl; }
      RUN(conv_gemm_tc(c, g));
      continue;
    }
    {
      ConvGemm g = make_gemm(d.layers[l].dil.f, s, b.y, C);
      g.e.mode = EPI_GATE; g.e.add = b.condall + (size_t)l * 2 * C; g.e.ld_add = L * 2 * C; g.e.out = b.zg; g.e.ldo = C;
      RUN(conv_gemm(c, g));
    }
    {
      ConvGemm g = make_gemm(d.layers[l].outp.f, s, b.zg, C);
      g.e.mode = EPI_RES_SKIP; g.e.C = C; g.e.res = b.x; g.e.ld_res = C; g.e.beta = 0.70710678118654752440f;
      g.e.out = b.x; g.e.ldo = C;
      if (l + 1 < L) { g.e.out2 = b.y; g.e.ldo2 = C; g.e.vec2 = dt + (size_t)(l + 1) * C; }
      g.e.skip = b.skip; g.e.ld_skip = C; g.e.skip_init = (l == 0);
      RUN(conv_gemm(c, g));
    }
  }
  return denoiser_heads(c, d, s, b);
}

bool denoiser_tc_ok(const Model& m, const Denoiser& d) { return m.use_tc && d.tc_ok; }
int alloc_denoiser(Ctx& c, const Denoiser& d, const SeqDev& s, bool tc, DenoiserBufs* b) {
  b->tc = tc;
  b->single_pass = false;
  b->condpre = nullptr;
  b->x = alloc_rows(c, s, d.C);
  b->y = b->zg = nullptr;
  b->yh = b->yl = b->zh = b->zl = b->ch = b->cl = nullptr;
  b->skh = b->skl = b->sh = b->sl = b->x80h = b->x80l = nullptr;
  b->condall = nullptr;
  b->tc_heads = tc && d.skip_tc.ok && d.out_tc.ok;
  if (b->tc_heads) {
    b->skh = alloc_half_rows(c, s, d.C);
    b->skl = alloc_half_rows(c, s, d.C);
    b->sh = alloc_half_rows(c, s, d.C);
    b->sl = alloc_half_rows(c, s, d.C);
    if (!d.ddiff && d.in_tc.ok) {
      b->x80h = alloc_half_rows(c, s, 128);
      b->x80l = alloc_half_rows(c, s, 128);
    }
  }
  if (tc) {
    b->yh = alloc_half_rows(c, s, d.C);
    b->yl = alloc_half_rows(c, s, d.C);
    b->zh = alloc_half_rows(c, s, d.C);
    b->zl = alloc_half_rows(c, s, d.C);
    b->ch = alloc_half_rows(c, s, 256);
    b->cl = alloc_half_rows(c, s, 256);
    // only valid rows are ever written or read (epilogues are row-bounded): no 4.6 GB memset for batch64
    b->condpre = alloc_rows(c, s, d.L * 2 * d.C, false);
  } else {
    b->y = alloc_rows(c, s, d.C);
    b->zg = alloc_rows(c, s, d.C);
    b->condall = alloc_rows(c, s, d.L * 2 * d.C, false);
  }
  // tensor-core heads: the fp32 skip accumulator is private to the RES_SKIP epilogue (the heads read the planes the last
  // layer writes), so it is kept chunk-tiled (every 32 x 32 epilogue chunk one contiguous 4 KB block; conv_gemm_tc.cuh)
  if (b->tc_heads) {
    const size_t n = (size_t)s.ntiles * TILE_M * d.C;
    b->skip = c.alloc<float>(n);  // fully written by layer 0 (skip_init) before it is read: no memset
  } else {
    b->skip = alloc_rows(c, s, d.C);
  }
  b->sbuf = b->tc_heads ? nullptr : alloc_rows(c, s, d.C);
  b->ld_head = b->tc_heads ? d.out_tc.N : ((d.out_dims + 3) & ~3);
  b->head = alloc_rows(c, s, b->ld_head);
  WS_OK(c);
  return 0;
}
// Tensor-core path: cond -> fp16 hi/lo planes (ch, cl) -> the step-invariant conditioner projection of all L layers at
// once, [rows, 256] x [256, L*2C], once per sampler call.  condpre is layer-major (row pitch 2C floats instead of L * 2C):
// matrix l is the GATE epilogue addend of layer l.
static int hoist_cond_tc(Ctx& c, const Denoiser& d, const SeqDev& s, const float* cond_g, __half* ch, __half* cl,
                         float* condpre, bool single_pass) {
  RUN(split_planes(c, cond_g, 256, s.rows, 256, 1.0f, ch, cl));
  GemmTC g = make_gemm_tc(d.cond_all_tc, s, ch, cl);
  g.single_pass = single_pass;
  g.e.out = condpre; g.e.ldo = d.L * 2 * d.C;
  g.e.out_nb = 2 * d.C; g.e.out_bs = (int64_t)s.rows * 2 * d.C;
  return conv_gemm_tc(c, g);
}
// Conditioner: the step-invariant projection of all L layers hoisted into one [rows, L*2C] buffer (tensor-core path:
// hoist_cond_tc; SIMT path: row-major, the layers side by side).
int prepare_cond(Ctx& c, const Denoiser& d, const SeqDev& s, const float* cond_g, DenoiserBufs& b) {
  if (b.tc) return hoist_cond_tc(c, d, s, cond_g, b.ch, b.cl, b.condpre, b.single_pass);
  ConvGemm g = make_gemm(d.cond_all, s, cond_g, 256);
  g.e.out = b.condall; g.e.ldo = d.L * 2 * d.C;
  return conv_gemm(c, g);
}

// a18 entry for one evaluation (mel): x80 [rows,80] guarded -> head
int mel_denoiser_eval(Ctx& c, const Denoiser& d, const SeqDev& s, int t, const float* x80, DenoiserBufs& b) {
  if (b.x80h) {  // tensor-core input projection: K padded 80 -> 128
    RUN(x80_planes(c, x80, s.rows, b.x80h, b.x80l));
    GemmTC g = make_gemm_tc(d.in_tc, s, b.x80h, b.x80l);
    g.single_pass = b.single_pass;
    g.e.bias = d.in_proj.bias; g.e.act = ACT_RELU;  // planes of y = relu(in_proj) + step bias only
    g.e.oh = b.yh; g.e.ol = b.yl; g.e.ldh = d.C; g.e.vec2 = d.dtab + (size_t)t * d.L * d.C;
    RUN(conv_gemm_tc(c, g));
    return denoiser_stack(c, d, s, t, b);
  }
  ConvGemm g = make_gemm(d.in_proj, s, x80, 80);
  g.e.act = ACT_RELU; g.e.out = b.x; g.e.ldo = d.C;
  g.e.vec2 = d.dtab + (size_t)t * d.L * d.C;
  if (b.tc) { g.e.out2_h = b.yh; g.e.out2_l = b.yl; g.e.ldh = d.C; }
  else { g.e.out2 = b.y; g.e.ldo2 = d.C; }
  RUN(conv_gemm(c, g));
  return denoiser_stack(c, d, s, t, b);
}

// Reverse steps of the mel sampler: hparams['K_step'] (DiffusionDecoder.forward's t = self.K_step,
// shallow_diffusion_tts.py:297-304), set by ssb_model_set_mel_k_step; 0 follows the schedule's T.  The reference would
// index past its schedule buffers with K > T, so that is an error here.
static int mel_k_step(const Model& m, int* K) {
  const int T = m.melnet.T;
  *K = m.mel_k_step > 0 ? m.mel_k_step : T;
  SSB_CHECK(*K <= T, "mel sampler: K_step " + std::to_string(*K) + " (ssb_model_set_mel_k_step) exceeds the schedule's T " +
                         std::to_string(T));
  return 0;
}

// x_K of the mel sampler.  DiffSinger: q_sample(norm_spec(coarse), K-1) on the T-step schedule
// (shallow_diffusion_tts.py:298-302); ProDiff: randn (prodiff.py:214-216), no coarse mel.  Both draw block 0 of the
// injected noise, or Philox stream_mel_xt().
static int mel_init(Ctx& c, const Model& m, const SeqDev& s, const float* coarse_g, const float* noise, int K, float* xm) {
  const Denoiser& d = m.melnet;
  if (m.mel_decoder == SSB_MEL_DECODER_PRODIFF)
    return mel_q_sample(c, s, nullptr, 80, noise, nullptr, nullptr, 0.f, 0.f, xm, 80, s.rng, stream_mel_xt());
  const float sa = c.dry ? 0.f : d.gtab_h[(size_t)(K - 1) * 8 + 5], s1a = c.dry ? 0.f : d.gtab_h[(size_t)(K - 1) * 8 + 6];
  return mel_q_sample(c, s, coarse_g, 80, noise, m.spec_min, m.spec_max, sa, s1a, xm, 80, s.rng, stream_mel_xt());
}
// x_0 -> mel_out.  DiffSinger: denorm_spec (shallow_diffusion_tts.py:305,274-275); ProDiff: denorm_spec is the identity
// and mel_out is not masked (prodiff.py:221-222,228-229).
static int mel_finish(Ctx& c, const Model& m, const SeqDev& s, const float* xm, float* mel_tight) {
  if (m.mel_decoder == SSB_MEL_DECODER_PRODIFF) return unpack_rows(c, s, xm, 80, mel_tight, 80, 80);
  return mel_denorm(c, s, xm, 80, m.spec_min, m.spec_max, nullptr, mel_tight, 80);
}

// ------------------------------------------------------------------------------------------------
// Persistent samplers (sampler_tc.cu): all T reverse steps of a denoiser in one cooperative launch, driven by a table
// of GEMM phases (SPhase) over a table of tensor maps.  PersistentNet is one DiffNet's part of such a launch; the
// samplers add their own input and sampling phases around it.
struct PersistentNet {
  // fp16 hi/lo plane pairs: pl[i] (hi) and pl[i + 1] (lo), tensor maps mb + i and mb + i + 1
  enum { Y = 0, Z = 2, SKIP = 4, S = 6, NPL = 8 };  // y = x + step bias, gate output, finished skip sum, relu(skip_proj)
  const Denoiser* d = nullptr;
  float* x = nullptr;        // fp32 residual stream [rows, C]
  float* skip = nullptr;     // skip accumulator [rows, C]
  __half* pl[NPL] = {};      // [rows, C] each
  float* condpre = nullptr;  // hoisted conditioner projection (hoist_cond_tc)
  int mb = 0;                // index of the net's first tensor map
  // the net's maps from mb: its NPL activation planes, then (hi, lo) weights of dil.t and outp.t per layer, skip, out
  static int nmaps(int L) { return NPL + 4 * L + 4; }
  int w_layer(int l) const { return mb + NPL + 4 * l; }  // dil.t; outp.t at + 2
  int w_skip() const { return mb + NPL + 4 * d->L; }
  int w_out() const { return w_skip() + 2; }
};

// Allocates the net's buffers and hoists its conditioner projection, so that its gate phases contract K = 3C and add
// that projection in the epilogue.  single_pass: the hoisted projection's precision, that of the launch's GEMMs.
static int persistent_net_setup(Ctx& c, const Denoiser& d, const SeqDev& s, const float* cond_g, int mb, bool single_pass,
                                PersistentNet* p) {
  p->d = &d;
  p->mb = mb;
  p->x = alloc_rows(c, s, d.C);
  p->skip = alloc_rows(c, s, d.C);
  for (int i = 0; i < PersistentNet::NPL; ++i) p->pl[i] = alloc_half_rows(c, s, d.C);
  __half* ch = alloc_half_rows(c, s, 256);
  __half* cl = alloc_half_rows(c, s, 256);
  p->condpre = alloc_rows(c, s, d.L * 2 * d.C, false);
  WS_OK(c);
  return hoist_cond_tc(c, d, s, cond_g, ch, cl, p->condpre, single_pass);
}

// Writes the net's tensor maps into maps[p.mb, p.mb + nmaps(L)); activation boxes of 128 / cs rows, one cs-th of an
// M-tile per CTA of a cluster.
static int persistent_net_maps(const PersistentNet& p, const SeqDev& s, int cs, CUtensorMap* maps) {
  const Denoiser& d = *p.d;
  for (int i = 0; i < PersistentNet::NPL; ++i)
    if (make_act_map(&maps[p.mb + i], p.pl[i], s.rows, d.C, 128 / cs)) return -1;
  auto put = [&](int idx, const ConvTC& w) { maps[idx] = w.tm_hi[0]; maps[idx + 1] = w.tm_lo[0]; };
  for (int l = 0; l < d.L; ++l) {
    put(p.w_layer(l), d.layers[l].dil.t);
    put(p.w_layer(l) + 2, d.layers[l].outp.t);
  }
  put(p.w_skip(), d.skip_tc);
  put(p.w_out(), d.out_tc);
  return 0;
}

static SPhase sphase(int sync_after) {
  SPhase z;
  memset(&z, 0, sizeof(z));
  z.taps = 1; z.dil = 1; z.beta = 1.0f; z.sync_after = sync_after;
  return z;
}

// Appends the net's phases of reverse step t, from its input planes y (written by the caller's previous phase) to the
// s planes: L (gate, residual + skip) pairs, then skip_projection.  Every entry gets sync_after.
static void persistent_net_step(const PersistentNet& p, const SeqDev& s, int t, int sync_after, std::vector<SPhase>& ph) {
  using P = PersistentNet;
  const Denoiser& d = *p.d;
  const int C = d.C, L = d.L;
  const float* dt = d.dtab + (size_t)t * L * C;
  for (int l = 0; l < L; ++l) {
    SPhase a = sphase(sync_after);  // dilated conv (3 taps of y) + hoisted conditioner projection -> gate -> z planes
    a.a1 = p.mb + P::Y; a.w1 = p.w_layer(l); a.taps = 3; a.kchunks = C / 64;
    a.dil = d.layers[l].dil.t.dil; a.center = 1; a.N = 2 * C; a.NT = 2 * C / 64; a.mode = SP_GATE;
    a.bias = d.layers[l].bias_gate_tc; a.wscale = d.layers[l].dil.t.wscale; a.oh = p.pl[P::Z]; a.ol = p.pl[P::Z + 1]; a.ldh = C;
    a.add = p.condpre + (size_t)l * (size_t)s.rows * 2 * C; a.ld_add = 2 * C;
    ph.push_back(a);
    SPhase b = sphase(sync_after);  // 1x1 output projection -> residual stream, next layer's input planes, skip sum
    b.a1 = p.mb + P::Z; b.w1 = p.w_layer(l) + 2; b.kchunks = C / 64; b.N = 2 * C; b.NT = 2 * C / 64; b.mode = SP_RES_SKIP;
    b.bias = d.layers[l].outp.f.bias; b.wscale = d.layers[l].outp.t.wscale; b.res = p.x; b.ld_res = C; b.out = p.x; b.ldo = C; b.beta = 0.70710678118654752440f;
    if (l + 1 < L) { b.oh = p.pl[P::Y]; b.ol = p.pl[P::Y + 1]; b.ldh = C; b.vec2 = dt + (size_t)(l + 1) * C; }
    b.skip = p.skip; b.ld_skip = C; b.C = C; b.skip_init = (l == 0);
    if (l == L - 1) { b.sh = p.pl[P::SKIP]; b.sl = p.pl[P::SKIP + 1]; }
    ph.push_back(b);
  }
  SPhase q = sphase(sync_after);  // skip_projection (1/sqrt(L) folded into the weights, N padded) + ReLU -> s planes
  q.a1 = p.mb + P::SKIP; q.w1 = p.w_skip(); q.kchunks = C / 64; q.N = d.skip_tc.N; q.NT = d.skip_tc.N / 64;
  q.mode = SP_SKIPPROJ; q.bias = d.skip_bias_pad; q.wscale = d.skip_tc.wscale; q.oh = p.pl[P::S]; q.ol = p.pl[P::S + 1]; q.ldh = C; q.n_valid = C;
  ph.push_back(q);
}

// a18+a19, single launch: all K reverse steps (t = K-1 .. 0) of the mel DiffNet, K (2L + 3) phases.
static int run_mel_diffusion_persistent(Ctx& c, const Model& m, const SeqDev& s, const float* cond_g, const float* coarse_g,
                                        const float* noise, int K, float* mel_tight) {
  using P = PersistentNet;
  const Denoiser& d = m.melnet;
  const int C = d.C, L = d.L;
  const int CS = 4;  // cluster size along N: A tiles are TMA-multicast to the 4 CTAs that share an M-tile
  const size_t mk = c.mark();
  float* xm = alloc_rows(c, s, 80);
  P net;
  RUN(persistent_net_setup(c, d, s, cond_g, 0, m.mel_fp16, &net));
  __half* x80h = alloc_half_rows(c, s, 128);  // planes of x_t, K padded 80 -> 128
  __half* x80l = alloc_half_rows(c, s, 128);
  const int M_X80 = P::nmaps(L), W_IN = M_X80 + 2, nmaps = W_IN + 2;
  const int nph = K * (2 * L + 3);
  CUtensorMap* maps_dev = c.alloc<CUtensorMap>((size_t)nmaps);
  SPhase* ph_dev = c.alloc<SPhase>((size_t)nph);
  unsigned* ctr = c.alloc<unsigned>(4);
  WS_OK(c);
  const size_t per = (size_t)s.total * 80;
  RUN(mel_init(c, m, s, coarse_g, noise, K, xm));
  RUN(x80_planes(c, xm, s.rows, x80h, x80l));
  if (!c.dry) {
    std::vector<CUtensorMap> maps((size_t)nmaps);
    if (persistent_net_maps(net, s, CS, maps.data())) return -1;
    if (make_act_map(&maps[M_X80], x80h, s.rows, 128, 128 / CS)) return -1;
    if (make_act_map(&maps[M_X80 + 1], x80l, s.rows, 128, 128 / CS)) return -1;
    maps[W_IN] = d.in_tc.tm_hi[0]; maps[W_IN + 1] = d.in_tc.tm_lo[0];
    std::vector<SPhase> ph;
    ph.reserve((size_t)nph);
    for (int t = K - 1; t >= 0; --t) {
      SPhase q = sphase(1);  // input_projection + ReLU ; y = x + step bias of layer 0
      q.a1 = M_X80; q.w1 = W_IN; q.kchunks = 2; q.N = C; q.NT = C / 64; q.mode = SP_INPROJ; q.bias = d.in_proj.bias;
      q.wscale = d.in_tc.wscale;
      q.out = net.x; q.ldo = C; q.oh = net.pl[P::Y]; q.ol = net.pl[P::Y + 1]; q.ldh = C; q.vec2 = d.dtab + (size_t)t * L * C;
      ph.push_back(q);
      persistent_net_step(net, s, t, 1, ph);
      q = sphase(1);  // output_projection -> eps ; fused DDPM posterior step on x_t
      q.a1 = net.mb + P::S; q.w1 = net.w_out(); q.kchunks = C / 64; q.N = 256; q.NT = 4; q.mode = SP_MEL_SAMPLE;
      q.bias = d.out_bias_pad; q.wscale = d.out_tc.wscale; q.out = xm; q.ldo = 80; q.oh = x80h; q.ol = x80l; q.ldh = 128; q.tab = d.gtab + (size_t)t * 8;
      q.noise = noise ? noise + per * (size_t)(K - t) : nullptr; q.stream_id = stream_mel_step(t); q.n_valid = 80;
      q.no_clip = m.mel_decoder == SSB_MEL_DECODER_PRODIFF;
      ph.push_back(q);
    }
    SSB_CUDA(cudaMemcpyAsync(maps_dev, maps.data(), sizeof(CUtensorMap) * nmaps, cudaMemcpyHostToDevice, c.stream));
    SSB_CUDA(cudaMemcpyAsync(ph_dev, ph.data(), sizeof(SPhase) * nph, cudaMemcpyHostToDevice, c.stream));
    RUN(launch_sampler_tc(c, maps_dev, ph_dev, nph, s, 2 * C / 64, ctr, CS, m.mel_fp16));
  }
  RUN(mel_finish(c, m, s, xm, mel_tight));
  c.release(mk);
  return 0;
}

// a18+a19: DiffusionDecoder.forward(infer=True) (shallow_diffusion_tts.py:284-307), or on a ProDiff model
// ProDiffusion.forward(infer=True) (prodiff.py:204-222; coarse_g unused, pass null)
int run_mel_diffusion(Ctx& c, const Model& m, const SeqDev& s, const float* cond_g, const float* coarse_g,
                      const float* noise /*tight [(K+1), total, 80] or null*/, float* mel_tight, const Seq* host_seq) {
  const Denoiser& d = m.melnet;
  SSB_CHECK(d.T > 0, "mel schedule not set: call ssb_model_set_schedule(which=0)");
  int K = 0;
  RUN(mel_k_step(m, &K));
  // ssb_model_set_persistent_groups(1): utterances are independent, so the K x L loop runs per GROUP of consecutive
  // utterances of <= 48 row tiles (a contiguous slice of the guard-banded layout: the sub-batch simply aliases the big
  // buffers), each by the single-launch persistent kernel (BASELINE.json configs[4]: persistent-kernel vs per-step-launch
  // at batch 64).  Production (Philox) mode only - the injected-noise tensors are strided by the whole batch.  With one
  // seed for the call each group g is keyed seed + 0x9E3779B97F4A7C15 g and counts its own rows; per-utterance seeds
  // carry over as they are (philox.cuh, "Batch composition").
  if (host_seq && !noise && !c.dry && m.persistent_groups && m.persistent && s.ntiles > 48) {
    int b0 = 0;
    int64_t tight0 = 0;
    int gi = 0;
    auto tiles_of = [&](int b) { return (host_seq->len[b] + TILE_M - 1) / TILE_M; };
    while (b0 < host_seq->B) {
      int b1 = b0;
      int64_t fr = 0, nt = 0;
      while (b1 < host_seq->B && (b1 == b0 || nt + tiles_of(b1) <= 48)) {
        nt += tiles_of(b1);
        fr += host_seq->len[b1++];
      }
      std::vector<int32_t> offs((size_t)(b1 - b0) + 1, 0);
      for (int b = b0; b < b1; ++b) offs[(size_t)(b - b0) + 1] = offs[(size_t)(b - b0)] + host_seq->len[b];
      Seq q;
      q.build(offs.data(), b1 - b0);
      q.seed = host_seq->seed + 0x9E3779B97F4A7C15ull * (uint64_t)gi;
      q.utt_seeds = host_seq->utt_seeds ? host_seq->utt_seeds + b0 : nullptr;
      const size_t mkg = c.mark();
      SeqDev sg;
      RUN(upload_layout(c, q, 1, &sg));
      const int64_t row_off = (int64_t)host_seq->rs[b0] - GUARD;  // the sub-layout's row 0 inside the big buffers
      RUN(run_mel_diffusion(c, m, sg, cond_g + row_off * 256, coarse_g ? coarse_g + row_off * 80 : nullptr, nullptr,
                            mel_tight + tight0 * 80, nullptr));
      c.release(mkg);
      tight0 += fr;
      b0 = b1;
      ++gi;
    }
    return 0;
  }
  if (m.persistent && denoiser_tc_ok(m, d) && d.in_tc.ok && d.skip_tc.ok && d.out_tc.ok && s.ntiles <= 48 &&
      sampler_tc_max_ctas() > 0)
    return run_mel_diffusion_persistent(c, m, s, cond_g, coarse_g, noise, K, mel_tight);
  const size_t mk = c.mark();
  DenoiserBufs b;
  RUN(alloc_denoiser(c, d, s, denoiser_tc_ok(m, d), &b));
  b.single_pass = b.tc && m.mel_fp16;
  float* xm = alloc_rows(c, s, 80);
  WS_OK(c);
  RUN(prepare_cond(c, d, s, cond_g, b));
  const size_t per = (size_t)s.total * 80;
  const bool clip = m.mel_decoder != SSB_MEL_DECODER_PRODIFF;
  RUN(mel_init(c, m, s, coarse_g, noise, K, xm));
  for (int t = K - 1; t >= 0; --t) {
    RUN(mel_denoiser_eval(c, d, s, t, xm, b));
    const float* nz = noise ? noise + per * (size_t)(K - t) : nullptr;
    RUN(mel_p_sample(c, s, xm, 80, b.head, b.ld_head, nz, d.gtab + (size_t)t * 8, s.rng, stream_mel_step(t), clip));
  }
  RUN(mel_finish(c, m, s, xm, mel_tight));
  c.release(mk);
  return 0;
}

// f2 (SURVEY 8f): PLMS / PNDM sampler over the same denoiser (GaussianDiffusion.p_sample_plms + the pndm_speedup loop of
// GaussianDiffusion.forward, shallow_diffusion_tts.py:164-197,254-260): K / interval evaluations (+1 for the first step).
int run_mel_diffusion_plms(Ctx& c, const Model& m, const SeqDev& s, const float* cond_g, const float* coarse_g,
                           const float* q_noise /*tight [total, 80] or null*/, int interval, float* mel_tight) {
  const Denoiser& d = m.melnet;
  SSB_CHECK(m.mel_decoder == SSB_MEL_DECODER_DIFFSINGER,
            "plms: the PLMS sampler needs a DiffSinger model (the ProDiff sampler predicts x0, not eps)");
  SSB_CHECK(d.T > 0, "mel schedule not set: call ssb_model_set_schedule(which=0)");
  int K = 0;
  RUN(mel_k_step(m, &K));
  SSB_CHECK(interval >= 1 && interval < K, "plms: interval (pndm_speedup) must be in [1, K_step)");
  const size_t mk = c.mark();
  DenoiserBufs b;
  RUN(alloc_denoiser(c, d, s, denoiser_tc_ok(m, d), &b));
  b.single_pass = b.tc && m.mel_fp16;
  float* xm = alloc_rows(c, s, 80);
  float* xp = alloc_rows(c, s, 80);
  float* hist[3] = {alloc_rows(c, s, 80), alloc_rows(c, s, 80), alloc_rows(c, s, 80)};
  WS_OK(c);
  RUN(prepare_cond(c, d, s, cond_g, b));
  auto acp = [&](int t) { return c.dry ? 0.5f : d.gtab_h[(size_t)t * 8 + 7]; };
  RUN(mel_init(c, m, s, coarse_g, q_noise, K, xm));
  int nh = 0;  // predictions in the history; hist[(head + k) % 3] is the k-th newest
  int head = 0;
  int t0 = 0;
  for (int t = 0; t < K; t += interval) t0 = t;  // reversed(range(0, K, interval)) starts at the largest multiple below K
  for (int t = t0; t >= 0; t -= interval) {
    const int tp = t - interval > 0 ? t - interval : 0;
    RUN(mel_denoiser_eval(c, d, s, t, xm, b));
    PlmsArgs a;
    a.x = xm; a.eps = b.head; a.lde = b.ld_head; a.a_t = acp(t); a.a_prev = acp(tp);
    const int slot = (head + 2) % 3;  // overwritten by this step's eps: the oldest entry
    if (nh == 0) {
      // second-order start: trial step with eps, second evaluation at the trial point, average (:182-185)
      PlmsArgs p1 = a;
      p1.x_out = xp; p1.hist_out = hist[slot];  // eps is saved before the head buffer is overwritten by the 2nd evaluation
      RUN(plms_update(c, s, p1));
      RUN(mel_denoiser_eval(c, d, s, tp, xp, b));
      a.h1 = hist[slot]; a.w0 = 1.f; a.w1 = 1.f; a.den = 2.f;  // (eps + eps_prev) / 2 with eps_prev = current head
      a.x_out = xm; a.hist_out = nullptr;
      RUN(plms_update(c, s, a));
    } else {
      const float* h1 = hist[head];
      const float* h2 = hist[(head + 1) % 3];
      const float* h3 = hist[(head + 2) % 3];
      if (nh == 1) { a.h1 = h1; a.w0 = 3.f; a.w1 = -1.f; a.den = 2.f; }
      else if (nh == 2) { a.h1 = h1; a.h2 = h2; a.w0 = 23.f; a.w1 = -16.f; a.w2 = 5.f; a.den = 12.f; }
      else { a.h1 = h1; a.h2 = h2; a.h3 = h3; a.w0 = 55.f; a.w1 = -59.f; a.w2 = 37.f; a.w3 = -9.f; a.den = 24.f; }
      a.x_out = xm;
      // the oldest entry (h3's slot) receives eps; with nh >= 3 the same element is read (h3) and then written by one thread
      a.hist_out = hist[slot];
      RUN(plms_update(c, s, a));
    }
    head = slot;
    if (nh < 3) ++nh;
  }
  RUN(mel_denorm(c, s, xm, 80, m.spec_min, m.spec_max, nullptr, mel_tight, 80));
  c.release(mk);
  return 0;
}

// a13+a14 for BOTH F0 nets in one persistent launch: the agnostic and the specific sampler are independent
// (stylesinger.py:223-225), so each phase of the table carries two entries (one per net, no barrier between them).
static int run_f0_diffusion_pair_persistent(Ctx& c, const Model& m, const SeqDev& s, const float* cond0, const float* cond1,
                                            const float* lo, const float* hi, const float* const gnoise[2],
                                            const float* const unoise[2], float* const z[2], int32_t* const uv[2]) {
  using P = PersistentNet;
  const int C = m.f0net[0].C, L = m.f0net[0].L, T = m.f0net[0].T;
  const int CS = 2;
  const size_t mk = c.mark();
  P net[2];
  for (int n = 0; n < 2; ++n)
    RUN(persistent_net_setup(c, m.f0net[n], s, n == 0 ? cond0 : cond1, n * P::nmaps(L), false, &net[n]));
  const int nmaps = 2 * P::nmaps(L);
  const int nph = 2 * T * (2 * L + 2);
  CUtensorMap* maps_dev = c.alloc<CUtensorMap>((size_t)nmaps);
  SPhase* ph_dev = c.alloc<SPhase>((size_t)nph);
  unsigned* ctr = c.alloc<unsigned>(4);
  WS_OK(c);
  const size_t per = (size_t)s.total;
  for (int n = 0; n < 2; ++n) {
    const Denoiser& d = m.f0net[n];
    RUN(f0_init(c, s, z[n], uv[n], gnoise[n], s.rng, stream_f0_xt(n)));
    RUN(ddiff_input(c, s, z[n], uv[n], d.in_w, d.in_b, d.uv_emb, d.dtab + (size_t)(T - 1) * L * C, net[n].x, nullptr, C,
                    net[n].pl[P::Y], net[n].pl[P::Y + 1]));
  }
  if (!c.dry) {
    std::vector<CUtensorMap> maps((size_t)nmaps);
    std::vector<SPhase> seq[2];  // each net's phases in order; sync_after on net 1's only
    for (int n = 0; n < 2; ++n) {
      const Denoiser& d = m.f0net[n];
      if (persistent_net_maps(net[n], s, CS, maps.data())) return -1;
      for (int t = T - 1; t >= 0; --t) {
        persistent_net_step(net[n], s, t, n == 1, seq[n]);
        SPhase q = sphase(n == 1);  // output_projection -> (eps, logits) ; F0/UV step ; DDiffNet input of step t-1
        q.a1 = net[n].mb + P::S; q.w1 = net[n].w_out(); q.kchunks = C / 64; q.N = d.out_tc.N; q.NT = d.out_tc.N / 64;
        q.mode = SP_F0_SAMPLE; q.bias = d.out_bias_pad; q.wscale = d.out_tc.wscale; q.out = z[n]; q.uv = uv[n]; q.clip_lo = lo; q.clip_hi = hi;
        q.tab = d.gtab + (size_t)t * 8; q.tab2 = d.mtab + (size_t)t * 8; q.tstep = t; q.log_eps = m.log_eps;
        q.noise = gnoise[n] ? gnoise[n] + per * (size_t)(T - t) : nullptr;
        q.noise2 = unoise[n] ? unoise[n] + per * 2 * (size_t)(T - 1 - t) : nullptr;
        q.stream_id = stream_f0_gauss(n, t); q.stream2 = stream_f0_unif(n, t);
        q.has_next = t > 0; q.C = C; q.in_w = d.in_w; q.in_b = d.in_b; q.uv_emb = d.uv_emb; q.x_next = net[n].x;
        q.oh = net[n].pl[P::Y]; q.ol = net[n].pl[P::Y + 1]; q.ldh = C;
        q.vec2 = t > 0 ? d.dtab + (size_t)(t - 1) * L * C : nullptr;
        seq[n].push_back(q);
      }
    }
    // number of clusters the launcher will use: needed for the tile-group rotation of the second net
    int ncl = s.ntiles * (2 * (2 * C / 64) / CS);
    {
      const int cap = sampler_tc_max_clusters(CS);
      if (ncl > cap) ncl = cap;
      if (ncl < 1) ncl = 1;
    }
    // the nets' entries alternate, so each phase holds one of each; net 1's tile groups start where net 0's end, so
    // one phase pair spreads over all clusters
    std::vector<SPhase> ph;
    ph.reserve((size_t)nph);
    for (size_t i = 0; i < seq[0].size(); ++i) {
      ph.push_back(seq[0][i]);
      ph.push_back(seq[1][i]);
      ph.back().goff = (s.ntiles * (seq[0][i].NT / CS)) % ncl;
    }
    SSB_CUDA(cudaMemcpyAsync(maps_dev, maps.data(), sizeof(CUtensorMap) * nmaps, cudaMemcpyHostToDevice, c.stream));
    SSB_CUDA(cudaMemcpyAsync(ph_dev, ph.data(), sizeof(SPhase) * nph, cudaMemcpyHostToDevice, c.stream));
    RUN(launch_sampler_tc(c, maps_dev, ph_dev, nph, s, 2 * (2 * C / 64), ctr, CS, false));
  }
  c.release(mk);
  return 0;
}
static bool f0_pair_persistent_ok(const Model& m, const SeqDev& s) {
  if (!m.persistent || !m.use_tc || s.ntiles > 48 || sampler_tc_max_ctas() <= 0) return false;
  for (int n = 0; n < 2; ++n) {
    const Denoiser& d = m.f0net[n];
    if (!denoiser_tc_ok(m, d) || !d.skip_tc.ok || !d.out_tc.ok || d.T <= 0) return false;
  }
  return m.f0net[0].C == m.f0net[1].C && m.f0net[0].L == m.f0net[1].L && m.f0net[0].T == m.f0net[1].T;
}

// a13+a14: GaussianMultinomialDiffusion.sample (gaussian_multinomial_diffusion.py:921-942)
int run_f0_diffusion(Ctx& c, const Model& m, int which, const SeqDev& s, const float* cond_g, const float* lo,
                     const float* hi, const float* gnoise, const float* unoise, float* z, int32_t* uv) {
  const Denoiser& d = m.f0net[which];
  SSB_CHECK(d.T > 0, "f0 schedule not set: call ssb_model_set_schedule(which=1)");
  const size_t mk = c.mark();
  DenoiserBufs b;
  RUN(alloc_denoiser(c, d, s, denoiser_tc_ok(m, d), &b));
  RUN(prepare_cond(c, d, s, cond_g, b));
  const int T = d.T;
  const size_t per = (size_t)s.total;
  RUN(f0_init(c, s, z, uv, gnoise, s.rng, stream_f0_xt(which)));
  for (int t = T - 1; t >= 0; --t) {
    const float* dt = d.dtab + (size_t)t * d.L * d.C;
    RUN(ddiff_input(c, s, z, uv, d.in_w, d.in_b, d.uv_emb, dt, b.tc ? nullptr : b.x, b.y, d.C, b.yh, b.yl));
    RUN(denoiser_stack(c, d, s, t, b));
    F0StepArgs a;
    a.z = z; a.uv = uv; a.out3 = b.head; a.ld3 = b.ld_head; a.lo = lo; a.hi = hi;
    a.gnoise = gnoise ? gnoise + per * (size_t)(T - t) : nullptr;
    a.unoise = unoise ? unoise + per * 2 * (size_t)(T - 1 - t) : nullptr;
    a.gtab = d.gtab + (size_t)t * 8; a.mtab = d.mtab + (size_t)t * 8; a.t = t; a.log_eps = m.log_eps;
    a.rng = s.rng; a.gauss_stream = stream_f0_gauss(which, t); a.unif_stream = stream_f0_unif(which, t);
    RUN(f0_p_sample(c, s, a));
  }
  c.release(mk);
  return 0;
}

int run_f0_samplers(Ctx& c, const Model& m, const SeqDev& s, const float* cond0, const float* cond1, const float* lo,
                    const float* hi, const float* const gnoise[2], const float* const unoise[2], float* const z[2],
                    int32_t* const uv[2]) {
  if (f0_pair_persistent_ok(m, s)) return run_f0_diffusion_pair_persistent(c, m, s, cond0, cond1, lo, hi, gnoise, unoise, z, uv);
  // The two samplers are independent (stylesinger.py:223-225): run the second one on the model's auxiliary stream so
  // that their latency-bound dependent chains overlap.  Disjoint workspace regions.
  // Two streams only for small batches (latency-bound chains).  From ~8k frames on every GEMM fills the GPU on its
  // own, and the CTA-pair (cluster) kernels used there must not run concurrently with each other from two streams:
  // that combination hung the GPU in an earlier version of these kernels (root cause not isolated).
  const bool fork = !c.dry && m.aux_stream != nullptr && s.ntiles <= 64;
  if (fork) {
    SSB_CUDA(cudaEventRecord(m.ev_fork, c.stream));
    SSB_CUDA(cudaStreamWaitEvent(m.aux_stream, m.ev_fork, 0));
  }
  const size_t off0 = c.off;
  RUN(run_f0_diffusion(c, m, 0, s, cond0, lo, hi, gnoise[0], unoise[0], z[0], uv[0]));
  c.off = c.high;  // keep sampler 0's buffers alive: sampler 1 allocates above them
  {
    Ctx c2 = c;
    if (fork) c2.stream = m.aux_stream;
    RUN(run_f0_diffusion(c2, m, 1, s, cond1, lo, hi, gnoise[1], unoise[1], z[1], uv[1]));
    if (c2.high > c.high) c.high = c2.high;
    c.failed = c.failed || c2.failed;
  }
  if (fork) {
    SSB_CUDA(cudaEventRecord(m.ev_join, m.aux_stream));
    SSB_CUDA(cudaStreamWaitEvent(c.stream, m.ev_join, 0));
  }
  c.off = off0;
  return 0;
}

// ------------------------------------------------------------------------------------------------
// a20/a21: HifiGanGenerator.forward (hifigan_nsf.py:144-169)
// Stages whose channel counts are multiples of 64 run on the tensor-core kernel: every conv input is carried as
// fp16 hi/lo planes of leaky_relu(x) written by the producing epilogue (the reference applies leaky_relu before
// every conv), residuals / MRF accumulators stay fp32.  The narrow stages (C = 32, 16, 8) run their ResBlocks through a
// time-grouped [rows/g, 64] view of the same memory with repacked weights, g = 64 / C (pack.cu, pack_conv_grouped).
// ResBlock1 (hifigan_nsf.py:30-66): r = c2(lrelu(c1(lrelu(r)))) + r three times; ResBlock2 (:69-90): r = c(lrelu(r)) + r
// twice.  The last conv of each block adds into the MRF accumulator (x 1/nk on the last block).
int run_vocoder(Ctx& c, const Vocoder& v, const Seq& seq, const float* mel_tight, const float* f0_tight,
                const float* rand_ini, const float* src_noise, float* wav_tight) {
  const size_t mk0 = c.mark();
  int hop = 1;
  for (auto& st : v.stages) hop *= st.u;
  SeqDev s1, s256;
  RUN(upload_layout(c, seq, 1, &s1));
  RUN(upload_layout(c, seq, hop, &s256));
  float* mel = alloc_rows(c, s1, 80);
  float* f0g = alloc_rows(c, s1, 1);
  float* har = nullptr;
  WS_OK(c);
  RUN(pack_rows(c, s1, mel_tight, 80, mel, 80, 80));
  const bool nsf = v.nsf && f0_tight != nullptr;
  if (nsf) {
    RUN(pack_rows(c, s1, f0_tight, 1, f0g, 1, 1));
    har = alloc_rows(c, s256, 1);
    const size_t mk = c.mark();
    double* scratch = c.alloc<double>(nsf_scratch_doubles(s256));
    WS_OK(c);
    RUN(nsf_source(c, s1, s256, f0g, v.lin_w, v.lin_b, rand_ini, src_noise, har, scratch, hop, (float)v.cfg.sample_rate));
    c.release(mk);
  }
  const bool tc = v.use_tc && tc_available();
  const bool sp = tc && v.fp16;  // single-pass fp16 tensor-core GEMMs (ssb_vocoder_set_precision)
  int C = v.cfg.initial_channel;
  float* x = alloc_rows(c, s1, C);
  __half *pin_h = nullptr, *pin_l = nullptr;  // planes of leaky_relu(stage input), when the next ups runs on tensor cores
  const bool up0_tc = tc && !v.stages.empty() && v.stages[0].up.t.ok;
  if (up0_tc) {
    pin_h = alloc_half_rows(c, s1, C);
    pin_l = alloc_half_rows(c, s1, C);
  }
  WS_OK(c);
  {
    ConvGemm g = make_gemm(v.pre, s1, mel, 80);
    g.e.out = x; g.e.ldo = C;
    if (up0_tc) { g.e.out2_h = pin_h; g.e.out2_l = pin_l; g.e.ldh = C; g.e.plane_act = ACT_LRELU; g.e.plane_slope = 0.1f; }
    RUN(conv_gemm(c, g));
  }
  int rate = 1;
  SeqDev sin = s1;
  float* xin = x;
  for (size_t i = 0; i < v.stages.size(); ++i) {
    const VocStage& st = v.stages[i];
    const int Co = st.Cout;
    const int rate_out = rate * st.u;
    SeqDev so;
    RUN(upload_layout(c, seq, rate_out, &so));
    const bool up_tc = tc && st.up.t.ok && pin_h != nullptr;
    // grouped stage: [rows, C] is processed as [rows/g, 64] (same memory) with the time-grouped weight packing.  At C = 32
    // only on tensor cores (the FFMA GEMM takes the 32-channel convs as they are); at C = 16 and 8 on both paths
    // (ssb_vocoder_create_ex checked rate_out % g == 0 there).
    const bool grouped = st.g > 1 && rate_out % st.g == 0 && (st.g > 2 || (tc && st.res_tc));
    const int g = grouped ? st.g : 1;
    const bool res_tc = tc && st.res_tc && (st.g == 1 || grouped);
    SeqDev sw = so;
    const int Cw = g * Co;
    if (grouped) {
      RUN(upload_layout(c, seq, rate_out / g, &sw));
      sw.rows = so.rows / g;  // exactly the memory of the [so.rows, Co] buffers (TMA zero-fills beyond)
    }
    const bool next_up_tc = tc && i + 1 < v.stages.size() && v.stages[i + 1].up.t.ok;
    float* xu = alloc_rows(c, so, Co);
    float* r = alloc_rows(c, so, Co);
    float* acc = alloc_rows(c, so, Co);
    float* xt = nullptr;
    __half *px_h = nullptr, *px_l = nullptr, *pt_h = nullptr, *pt_l = nullptr, *pr_h = nullptr, *pr_l = nullptr;
    __half *pa_h = nullptr, *pa_l = nullptr;
    const bool rb2 = v.resblock == 2;  // ResBlock2 has no inner conv pair: no xt
    if (res_tc) {
      px_h = alloc_half_rows(c, so, Co); px_l = alloc_half_rows(c, so, Co);
      if (!rb2) { pt_h = alloc_half_rows(c, so, Co); pt_l = alloc_half_rows(c, so, Co); }
      pr_h = alloc_half_rows(c, so, Co); pr_l = alloc_half_rows(c, so, Co);
    } else if (!rb2) {
      xt = alloc_rows(c, so, Co);
    }
    if (next_up_tc) { pa_h = alloc_half_rows(c, so, Co); pa_l = alloc_half_rows(c, so, Co); }
    WS_OK(c);
    // fp16 planes of leaky_relu(v, 0.1), the pre-activation of the conv that consumes them, beside an epilogue's output
    auto lrelu_planes = [](Epi& e, __half* hi, __half* lo, int ld) {
      e.out2_h = hi; e.out2_l = lo; e.ldh = ld; e.plane_act = ACT_LRELU; e.plane_slope = 0.1f;
    };
    {  // x = ups[i](leaky_relu(x, 0.1))
      Epi e;
      e.out = xu; e.ldo = st.u * Co;
      if (res_tc && !nsf) lrelu_planes(e, px_h, px_l, st.u * Co);
      RUN(run_dense(c, st.up, up_tc, sin, {xin, C, pin_h, pin_l, ACT_LRELU, 0.1f}, e, sp));
    }
    if (nsf) RUN(noise_conv_add(c, so, s256, xu, Co, Co, har, st.nc_w, st.nc_b, st.nc_s, res_tc ? px_h : nullptr, px_l, 0.1f, st.nc_wt));
    const int nconv = rb2 ? 2 : 3;
    for (int j = 0; j < v.nk; ++j) {  // MRF: mean of the resblocks
      const float* rin = xu;
      const __half *rin_h = px_h, *rin_l = px_l;
      for (int mI = 0; mI < nconv; ++mI) {
        const bool last = (mI == nconv - 1);
        const bool lastj = (j == v.nk - 1);
        if (!rb2) {  // xt = c1(leaky_relu(r)) ; on tensor cores only leaky_relu(xt) is ever consumed -> planes only
          Epi e;
          if (res_tc) lrelu_planes(e, pt_h, pt_l, Cw);
          else { e.out = xt; e.ldo = Cw; }
          RUN(run_dense(c, st.rb[j].c1[mI], res_tc, sw, {rin, Cw, rin_h, rin_l, ACT_LRELU, 0.1f}, e, sp));
        }
        Epi e;  // ResBlock1: r = c2(leaky_relu(xt)) + r ; ResBlock2: r = c(leaky_relu(r)) + r
        e.res = rin; e.ld_res = Cw;
        if (!last) {
          e.out = r; e.ldo = Cw;
          if (res_tc) lrelu_planes(e, pr_h, pr_l, Cw);
        } else {
          e.out = acc; e.ldo = Cw; e.accum = (j > 0); e.gamma = lastj ? 1.0f / (float)v.nk : 1.0f;
          if (lastj && next_up_tc) lrelu_planes(e, pa_h, pa_l, Cw);
        }
        if (rb2) RUN(run_dense(c, st.rb[j].c1[mI], res_tc, sw, {rin, Cw, rin_h, rin_l, ACT_LRELU, 0.1f}, e, sp));
        else RUN(run_dense(c, st.rb[j].c2[mI], res_tc, sw, {xt, Cw, pt_h, pt_l, ACT_LRELU, 0.1f}, e, sp));
        rin = r; rin_h = pr_h; rin_l = pr_l;
      }
    }
    xin = acc; sin = so; C = Co; rate = rate_out;
    pin_h = pa_h; pin_l = pa_l;
  }
  if (v.post.N == 1 && C % 4 == 0 && (size_t)((256 + v.post.taps - 1) * (C + 1) + v.post.taps * C) * 4 <= 48 * 1024) {
    // N = 1: dedicated windowed reduction (leaky_relu 0.01 -> conv_post -> tanh in one pass over x)
    RUN(conv_post_tanh(c, sin, xin, C, C, v.post.taps, v.post.center, v.post.W, v.post.Npad, v.post.bias, 0.01f, wav_tight));
  } else {
    float* y = alloc_rows(c, sin, 4);
    WS_OK(c);
    ConvGemm g = make_gemm(v.post, sin, xin, C);
    g.a_act = ACT_LRELU; g.a_slope = 0.01f;  // F.leaky_relu default slope (hifigan_nsf.py:165)
    g.e.out = y; g.e.ldo = 4;
    RUN(conv_gemm(c, g));
    RUN(tanh_out(c, sin, y, 4, wav_tight));
  }
  c.release(mk0);
  return 0;
}

}  // namespace ssb
