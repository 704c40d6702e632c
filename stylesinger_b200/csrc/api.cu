// extern "C" boundary (include/stylesinger_b200.h) + the whole-model driver.
#include <stdlib.h>
#include <string.h>

#include "stages.cuh"

struct ssb_model { ssb::Model m; };
struct ssb_vocoder { ssb::Vocoder v; };

namespace ssb {

// project per-utterance vectors (spk_embed_proj / emo_embed_proj, stylesinger.py:130-132)
static int project_vec(Ctx& c, const Conv& w, const float* in_tight, int B, float* out_tight) {
  Seq s1;
  int32_t offs[2] = {0, B};
  s1.build(offs, 1);
  const size_t mk = c.mark();
  SeqDev sd;
  RUN(upload_layout(c, s1, 1, &sd));
  float* a = alloc_rows(c, sd, 256);
  float* o = alloc_rows(c, sd, 256);
  WS_OK(c);
  RUN(pack_rows(c, sd, in_tight, 256, a, 256, 256));
  ConvGemm g = make_gemm(w, sd, a, 256);
  g.e.out = o; g.e.ldo = 256;
  RUN(conv_gemm(c, g));
  RUN(unpack_rows(c, sd, o, 256, out_tight, 256, 256));
  c.release(mk);
  return 0;
}

// spk_embed_proj(spk_id) of a use_spk_id model (Embedding(num_spk + 1, 256), fs2.py:37-38): the ids (host, checked by the
// caller) go into a one-sequence layout of B rows and pitch_embed's row gather reads the table rows
static int gather_spk(Ctx& c, const Model& m, const int32_t* ids_host, int B, float* out_tight) {
  Seq s1;
  int32_t offs[2] = {0, B};
  s1.build(offs, 1);
  const size_t mk = c.mark();
  SeqDev sd;
  RUN(upload_layout(c, s1, 1, &sd));
  int32_t* idx = alloc_rows_i32(c, sd);
  float* o = alloc_rows(c, sd, 256);
  WS_OK(c);
  if (!c.dry) SSB_CUDA(cudaMemcpyAsync(idx + s1.rs[0], ids_host, sizeof(int32_t) * B, cudaMemcpyHostToDevice, c.stream));
  RUN(embed_rows(c, sd, idx, m.spk_tab, m.spk_rows, 1.0f, o, 256, 256, 0));
  RUN(unpack_rows(c, sd, o, 256, out_tight, 256, 256));
  c.release(mk);
  return 0;
}

// StyleSinger.forward(infer=True) (stylesinger.py:119-187); durations_only stops after add_dur.
int run_acoustic(Ctx& c, const Model& m, const ssb_acoustic_inputs& in, const ssb_acoustic_outputs& out,
                 bool durations_only, int32_t* dur_out, float* logdur_out, const uint64_t* utt_seeds) {
  const int H = 256, B = in.B;
  const bool emo_on = m.sw.emo != 0, style_on = m.sw.style != 0;
  SSB_CHECK(B >= 1 && in.ph_offsets && (in.ref_offsets || !style_on), "acoustic: bad batch description");
  // switched-off modules (ssb_model_create_ex3): their outputs do not exist
  SSB_CHECK(emo_on || !out.emo_proj, "acoustic: a model without emo (switch emo = 0) has no emo_proj");
  SSB_CHECK(style_on || (!out.style && !out.rq_codes),
            "acoustic: a model without style (switch style = 0) has no style / rq_codes");
  SSB_CHECK(durations_only || in.frame_offsets, "acoustic: frame_offsets required");
  SSB_CHECK(durations_only || in.mel2ph || in.dur, "acoustic: need mel2ph or dur");
  SSB_CHECK(m.mel_decoder != SSB_MEL_DECODER_PRODIFF || (!out.coarse_mel && !out.diff_cond),
            "acoustic: a ProDiff model has no coarse_mel / diff_cond (decoder_inp is the sampler's condition)");
  SSB_CHECK(m.f0_gen != SSB_F0_GEN_CONV || (!in.f0_gauss_noise[0] && !in.f0_gauss_noise[1] && !in.f0_unif_noise[0] &&
                                            !in.f0_unif_noise[1]),
            "acoustic: a model with the conv F0 generator draws no F0 noise (f0_gauss_noise / f0_unif_noise must be NULL)");
  const bool fft = m.mel_decoder == SSB_MEL_DECODER_FFT;
  SSB_CHECK(!fft || !out.diff_cond, "acoustic: a model with the FFT mel decoder has no diff_cond (there is no ln_proj)");
  SSB_CHECK(!fft || !in.mel_noise, "acoustic: a model with the FFT mel decoder draws no mel noise (mel_noise must be NULL)");
  if (m.spk_id) {  // use_spk_id: every id must index the table (checked here, before anything is launched)
    SSB_CHECK(in.spk_ids, "acoustic: a model created with use_spk_id needs spk_ids (host [B] speaker ids)");
    for (int b = 0; b < B; ++b)
      SSB_CHECK(in.spk_ids[b] >= 0 && in.spk_ids[b] < m.spk_rows,
                "acoustic: spk_ids[" + std::to_string(b) + "] = " + std::to_string(in.spk_ids[b]) + " is outside [0, " +
                    std::to_string(m.spk_rows) + ") (the rows of spk_embed_proj.weight)");
  }
  Seq qp, qr, qf;
  qp.build(in.ph_offsets, B);
  if (style_on) qr.build(in.ref_offsets, B);
  SSB_CHECK(qp.maxlen + 2 <= m.pos_rows && (!style_on || qr.maxlen + 2 <= m.pos_rows), "sequence longer than __pos_table");
  SeqDev sp, sr, sf;
  RUN(upload_layout(c, qp, 1, &sp));
  if (style_on) RUN(upload_layout(c, qr, 1, &sr));
  int32_t* tok = alloc_rows_i32(c, sp);
  int32_t* note = alloc_rows_i32(c, sp);
  int32_t* ntype = alloc_rows_i32(c, sp);
  float* ndur = alloc_rows(c, sp, 1);
  float* srcmask = alloc_rows(c, sp, 1);
  float* enc = alloc_rows(c, sp, H);
  float* spk = c.alloc<float>((size_t)B * H);
  float* emo = emo_on ? c.alloc<float>((size_t)B * H) : nullptr;  // null: combine_rows / concat_cond skip it
  WS_OK(c);
  RUN(pack_rows_i32(c, sp, in.txt_tokens, tok));
  RUN(pack_rows_i32(c, sp, in.note, note));
  RUN(pack_rows_i32(c, sp, in.note_type, ntype));
  RUN(pack_rows(c, sp, in.note_dur, 1, ndur, 1, 1));
  if (m.spk_id)
    RUN(gather_spk(c, m, in.spk_ids, B, spk));
  else
    RUN(project_vec(c, m.spk_proj, in.spk_embed, B, spk));
  if (emo_on) RUN(project_vec(c, m.emo_proj, in.emo_embed, B, emo));
  if (out.spk_proj && !c.dry) SSB_CUDA(cudaMemcpyAsync(out.spk_proj, spk, sizeof(float) * B * H, cudaMemcpyDeviceToDevice, c.stream));
  if (out.emo_proj && !c.dry) SSB_CUDA(cudaMemcpyAsync(out.emo_proj, emo, sizeof(float) * B * H, cudaMemcpyDeviceToDevice, c.stream));
  RUN(run_encoder(c, m, sp, tok, note, ntype, ndur, srcmask, enc));
  if (out.encoder_out) RUN(unpack_rows(c, sp, enc, H, out.encoder_out, H, H));

  if (durations_only) {
    float* dinp = alloc_rows(c, sp, H);
    float* logdur = alloc_rows(c, sp, 1);
    int32_t* dur = alloc_rows_i32(c, sp);
    WS_OK(c);
    CombineArgs a;  // dur_inp = (encoder_out + spk [+ emo]) * src_nonpadding (stylesinger.py:134-138)
    a.m[0] = enc; a.ldm[0] = H; a.v[0] = spk; a.v[1] = emo; a.rowmask = srcmask; a.out = dinp; a.ldo = H; a.C = H;
    RUN(combine_rows(c, sp, a));
    RUN(run_duration_predictor(c, m, sp, dinp, srcmask, logdur, dur));
    if (dur_out) RUN(unpack_rows_i32(c, sp, dur, dur_out));
    if (logdur_out) RUN(unpack_rows(c, sp, logdur, 1, logdur_out, 1, 1));
    return 0;
  }

  qf.build(in.frame_offsets, B);
  qf.seed = in.seed;
  qf.utt_seeds = utt_seeds;
  SSB_CHECK(qf.maxlen + 2 <= m.pos_rows, "frame sequence longer than __pos_table");
  RUN(upload_layout(c, qf, 1, &sf));
  int32_t* mel2ph = alloc_rows_i32(c, sf);
  int32_t* midi = alloc_rows_i32(c, sf);
  float* tgt = alloc_rows(c, sf, 1);
  float* dec0 = alloc_rows(c, sf, H);
  float* ref = style_on ? alloc_rows(c, sr, 80) : nullptr;
  float* reff0 = style_on ? alloc_rows(c, sr, 1) : nullptr;
  float* style = style_on ? alloc_rows(c, sf, H) : nullptr;  // null: combine_rows / concat_cond skip it
  int32_t* codes = style_on ? alloc_rows_i32(c, sr, m.hp.rq_depth) : nullptr;
  WS_OK(c);
  if (in.mel2ph) {
    RUN(pack_rows_i32(c, sf, in.mel2ph, mel2ph));
  } else {
    int32_t* dur = alloc_rows_i32(c, sp);
    WS_OK(c);
    RUN(pack_rows_i32(c, sp, in.dur, dur));
    RUN(length_regulate(c, sf, sp, dur, mel2ph));
  }
  if (out.mel2ph) RUN(unpack_rows_i32(c, sf, mel2ph, out.mel2ph));
  RUN(expand_states(c, sf, sp, mel2ph, enc, H, dec0, H, H, note, midi, tgt));
  if (style_on) {  // get_style (stylesinger.py:149-151)
    RUN(pack_rows(c, sr, in.ref_mels, 80, ref, 80, 80));
    RUN(pack_rows(c, sr, in.ref_f0, 1, reff0, 1, 1));
    RUN(run_style(c, m, sf, sr, dec0, ref, reff0, style, codes, nullptr));
    if (out.style) RUN(unpack_rows(c, sf, style, H, out.style, H, H));
    if (out.rq_codes) {
      // codes are [rows, depth] int32: unpack column by column through the i32 row copier
      for (int d = 0; d < m.hp.rq_depth; ++d) RUN(unpack_cols_i32(c, sr, codes, m.hp.rq_depth, d, out.rq_codes));
    }
  }

  // ---- pitch (inpaint_pitch, stylesinger.py:216-247)
  float* pitch_pred = alloc_rows(c, sf, 2);
  float* f0_denorm = alloc_rows(c, sf, 1);
  int32_t* pitch = alloc_rows_i32(c, sf);
  float* f0_in = nullptr;
  float* uv_in = nullptr;
  WS_OK(c);
  if (m.f0_gen == SSB_F0_GEN_CONV) {
    // f0_gen 'conv' (:223-236): both PitchPredictors always run (teacher-forced f0 only replaces f0 / uv); no MIDI band,
    // no noise
    const size_t mk = c.mark();
    float* cond = alloc_rows(c, sf, H);
    float* cond2 = alloc_rows(c, sf, H);
    float* pa = alloc_rows(c, sf, 2);
    float* ps = alloc_rows(c, sf, 2);
    WS_OK(c);
    if (in.f0) {
      f0_in = alloc_rows(c, sf, 1);
      uv_in = alloc_rows(c, sf, 1);
      WS_OK(c);
      RUN(pack_rows(c, sf, in.f0, 1, f0_in, 1, 1));
      if (in.uv) RUN(pack_rows(c, sf, in.uv, 1, uv_in, 1, 1));
    }
    {
      CombineArgs a;  // pitch_inp_domain_agnostic = decoder_inp * tgt_nonpadding (:156)
      a.m[0] = dec0; a.ldm[0] = H; a.rowmask = tgt; a.out = cond; a.ldo = H; a.C = H;
      RUN(combine_rows(c, sf, a));
    }
    {
      CombineArgs a;  // (decoder_inp + spk [+ emo] [+ style]) * tgt_nonpadding (:157-163)
      a.m[0] = dec0; a.ldm[0] = H; a.m[1] = style; a.ldm[1] = H; a.v[0] = spk; a.v[1] = emo;
      a.rowmask = tgt; a.out = cond2; a.ldo = H; a.C = H;
      RUN(combine_rows(c, sf, a));
    }
    // the FFT decoder's rule for its FFN GEMMs: long batches on the tensor-core kernel
    const bool tc = long_batch_tc(m, sf);
    RUN(run_pitch_predictor(c, m, 0, sf, cond, pa, tc));
    RUN(run_pitch_predictor(c, m, 1, sf, cond2, ps, tc));
    PitchGlueConvArgs pg;
    pg.pa = pa; pg.ps = ps; pg.mel2ph = mel2ph;
    pg.f0_in = f0_in; pg.uv_in = in.uv ? uv_in : nullptr;
    pg.pitch_pred = pitch_pred; pg.f0_denorm = f0_denorm; pg.pitch = pitch;
    RUN(pitch_glue_conv(c, sf, pg));
    c.release(mk);
  } else {
    const size_t mk = c.mark();
    float* za = alloc_rows(c, sf, 1);
    float* zs = alloc_rows(c, sf, 1);
    int32_t* uva = alloc_rows_i32(c, sf);
    int32_t* uvs = alloc_rows_i32(c, sf);
    WS_OK(c);
    if (in.f0) {
      // teacher forcing: the reference skips the samplers when f0 is passed (add_gmdiff_pitch :251-254)
      f0_in = alloc_rows(c, sf, 1);
      uv_in = alloc_rows(c, sf, 1);
      WS_OK(c);
      RUN(pack_rows(c, sf, in.f0, 1, f0_in, 1, 1));
      if (in.uv) RUN(pack_rows(c, sf, in.uv, 1, uv_in, 1, 1));
    } else {
      float* lo = alloc_rows(c, sf, 1);
      float* hi = alloc_rows(c, sf, 1);
      float* cond = alloc_rows(c, sf, H);
      float* cond2 = alloc_rows(c, sf, H);
      WS_OK(c);
      RUN(midi_clip_band(c, sf, midi, lo, hi));
      {
        CombineArgs a;  // pitch_inp_domain_agnostic = decoder_inp * tgt_nonpadding (:156)
        a.m[0] = dec0; a.ldm[0] = H; a.rowmask = tgt; a.out = cond; a.ldo = H; a.C = H;
        RUN(combine_rows(c, sf, a));
      }
      {
        CombineArgs a;  // (decoder_inp + spk [+ emo] [+ style]) * tgt_nonpadding (:157-163)
        a.m[0] = dec0; a.ldm[0] = H; a.m[1] = style; a.ldm[1] = H; a.v[0] = spk; a.v[1] = emo;
        a.rowmask = tgt; a.out = cond2; a.ldo = H; a.C = H;
        RUN(combine_rows(c, sf, a));
      }
      float* zz[2] = {za, zs};
      int32_t* uu[2] = {uva, uvs};
      RUN(run_f0_samplers(c, m, sf, cond, cond2, lo, hi, in.f0_gauss_noise, in.f0_unif_noise, zz, uu));
    }
    PitchGlueArgs pg;
    pg.za = za; pg.uva = uva; pg.zs = zs; pg.uvs = uvs; pg.midi = midi; pg.mel2ph = mel2ph;
    pg.f0_in = f0_in; pg.uv_in = in.uv ? uv_in : nullptr;
    pg.pitch_pred = pitch_pred; pg.f0_denorm = f0_denorm; pg.pitch = pitch;
    RUN(pitch_glue(c, sf, pg));
    c.release(mk);
  }
  if (out.pitch_pred) RUN(unpack_rows(c, sf, pitch_pred, 2, out.pitch_pred, 2, 2));
  if (out.f0_denorm) RUN(unpack_rows(c, sf, f0_denorm, 1, out.f0_denorm, 1, 1));

  // ---- decoder input (:165-172)
  float* dec = alloc_rows(c, sf, H);
  float* pemb = alloc_rows(c, sf, H);
  WS_OK(c);
  RUN(embed_rows(c, sf, pitch, m.pitch_emb, 300, 1.0f, pemb, H, H, 0));
  {
    CombineArgs a;  // (decoder_inp + spk + pitch_embed [+ emo] [+ style]) * tgt_nonpadding (:167-172)
    a.m[0] = dec0; a.ldm[0] = H; a.m[1] = pemb; a.ldm[1] = H; a.m[2] = style; a.ldm[2] = H;
    a.v[0] = spk; a.v[1] = emo; a.rowmask = tgt; a.out = dec; a.ldo = H; a.C = H;
    RUN(combine_rows(c, sf, a));
  }
  if (out.decoder_inp) RUN(unpack_rows(c, sf, dec, H, out.decoder_inp, H, H));

  if (m.mel_decoder == SSB_MEL_DECODER_PRODIFF) {
    // ProDiff (stylesinger.py:176-177): ret = diff_decoder(decoder_inp, ...) - no FFT decoder, mel_out, ln_proj or coarse
    // mel, and no pndm_speedup (ProDiffusion.forward never reads it)
    if (!in.skip_mel_diffusion) {
      SSB_CHECK(out.mel_out != nullptr, "acoustic: mel_out required");
      RUN(run_mel_diffusion(c, m, sf, dec, nullptr, in.mel_noise, out.mel_out, &qf));
    }
    return 0;
  }

  if (fft) {
    // decoder 'fft' (stylesinger.py:185-186): ret['mel_out'] = run_decoder(decoder_inp) = mel_out(decoder(x)) *
    // tgt_nonpadding (fs2.py:233-237) - the DiffSinger path's coarse mel, with no ln_proj and no diffusion after it
    float* mel = alloc_rows(c, sf, 80);
    float* xd = alloc_rows(c, sf, H);
    WS_OK(c);
    RUN(run_fft_decoder(c, m, sf, dec, xd, long_batch_tc(m, sf)));
    ConvGemm g = make_gemm(m.mel_out, sf, xd, H);
    g.e.rowmask = tgt; g.e.out = mel; g.e.ldo = 80;
    RUN(conv_gemm(c, g));
    if (out.mel_out) RUN(unpack_rows(c, sf, mel, 80, out.mel_out, 80, 80));
    if (out.coarse_mel) RUN(unpack_rows(c, sf, mel, 80, out.coarse_mel, 80, 80));
    return 0;
  }

  // ---- FFT decoder + mel_out (fs2.py:233-237, tts_modules.py:281-306)
  float* coarse = alloc_rows(c, sf, 80);
  float* cond = alloc_rows(c, sf, H);
  WS_OK(c);
  {
    const size_t mk = c.mark();
    float* xd = alloc_rows(c, sf, H);
    WS_OK(c);
    // long batches: the decoder's FFN GEMMs on the tensor-core kernel (short ones stay on the fp32 FFMA path, which is
    // what the reference-golden parity tests pin)
    RUN(run_fft_decoder(c, m, sf, dec, xd, long_batch_tc(m, sf)));
    {
      ConvGemm g = make_gemm(m.mel_out, sf, xd, H);
      g.e.rowmask = tgt; g.e.out = coarse; g.e.ldo = 80;
      RUN(conv_gemm(c, g));
    }
    // run_diffsinger: g = ln_proj(cat[coarse, [decoder_inp], spk, [emo], [style]]) (stylesinger.py:313-327)
    float* cat = alloc_rows(c, sf, m.cond_width);
    WS_OK(c);
    RUN(concat_cond(c, sf, coarse, m.sw.use_txt_cond ? dec : nullptr, spk, emo, style, cat, m.cond_width));
    {
      ConvGemm g = make_gemm(m.ln_proj, sf, cat, m.cond_width);
      g.e.out = cond; g.e.ldo = H;
      RUN(conv_gemm(c, g));
    }
    c.release(mk);
  }
  if (out.coarse_mel) RUN(unpack_rows(c, sf, coarse, 80, out.coarse_mel, 80, 80));
  if (out.diff_cond) RUN(unpack_rows(c, sf, cond, H, out.diff_cond, H, H));
  if (!in.skip_mel_diffusion) {
    SSB_CHECK(out.mel_out != nullptr, "acoustic: mel_out required");
    if (in.pndm_speedup > 0)  // PLMS: mel_noise, when given, supplies only the q_sample draw (its first [sumF, 80] block)
      RUN(run_mel_diffusion_plms(c, m, sf, cond, coarse, in.mel_noise, in.pndm_speedup, out.mel_out));
    else
      RUN(run_mel_diffusion(c, m, sf, cond, coarse, in.mel_noise, out.mel_out, &qf));
  }
  return 0;
}

int denoiser_eval_api(Ctx& c, const Model& m, int which, const SeqDev& s, const float* x_tight, const int32_t* uv_tight,
                      int t, const float* cond_tight, float* out_tight) {
  const Denoiser& d = which == 0 ? m.melnet : m.f0net[which - 1];
  SSB_CHECK(d.T > 0, "denoiser_eval: schedule not set");
  float* cond = alloc_rows(c, s, 256);
  DenoiserBufs b;
  RUN(alloc_denoiser(c, d, s, denoiser_tc_ok(m, d), &b));
  b.single_pass = b.tc && which == 0 && m.mel_fp16;  // the mel net follows ssb_model_set_mel_precision, the F0 nets stay split
  RUN(pack_rows(c, s, cond_tight, 256, cond, 256, 256));
  RUN(prepare_cond(c, d, s, cond, b));
  if (which == 0) {
    float* x80 = alloc_rows(c, s, 80);
    WS_OK(c);
    RUN(pack_rows(c, s, x_tight, 80, x80, 80, 80));
    RUN(mel_denoiser_eval(c, d, s, t, x80, b));
  } else {
    float* z = alloc_rows(c, s, 1);
    int32_t* uv = alloc_rows_i32(c, s);
    WS_OK(c);
    RUN(pack_rows(c, s, x_tight, 1, z, 1, 1));
    RUN(pack_rows_i32(c, s, uv_tight, uv));
    const float* dt = d.dtab + (size_t)t * d.L * d.C;
    RUN(ddiff_input(c, s, z, uv, d.in_w, d.in_b, d.uv_emb, dt, b.tc ? nullptr : b.x, b.y, d.C, b.yh, b.yl));
    RUN(denoiser_stack(c, d, s, t, b));
  }
  RUN(unpack_rows(c, s, b.head, b.ld_head, out_tight, d.out_dims, d.out_dims));
  return 0;
}

}  // namespace ssb

// ================================================================================================
using namespace ssb;

static int to_map(const ssb_tensor_desc* t, int n, TensorMap* tm) {
  for (int i = 0; i < n; ++i) {
    SSB_CHECK(t[i].name && t[i].data && t[i].ndim >= 1 && t[i].ndim <= 4, "bad tensor descriptor");
    HostTensor h;
    h.data = t[i].data;
    for (int d = 0; d < t[i].ndim; ++d) h.shape.push_back(t[i].shape[d]);
    tm->t[t[i].name] = h;
  }
  return 0;
}
static Ctx make_ctx(void* ws, size_t bytes, void* stream, bool dry = false) {
  Ctx c;
  c.base = (char*)ws; c.cap = bytes; c.stream = (cudaStream_t)stream; c.dry = dry;
  return c;
}

// ---- one dense GEMM at unit-test granularity (ssb_op_gemm) ---------------------------------------------------------------
struct OpWeights {  // the call's packed weights, freed with the pool when the call returns
  DevicePool pool;
  Conv cv;
  ConvTC ct;
};

// Packs the host weights for the call's path.  A conv whose taps reach past the guard band would read the neighbouring
// utterance (or, for the first one, whatever lies before the buffer), so it is refused here, before anything is launched.
static int op_pack(const ssb_op_gemm_args& a, OpWeights* w) {
  SSB_CHECK(a.path == 0 || a.path == 1, "op_gemm: path must be 0 (fp32 FFMA) or 1 (tensor cores)");
  SSB_CHECK(a.single_pass == 0 || (a.single_pass == 1 && a.path == 1),
            "op_gemm: single_pass must be 0, or 1 on path 1 (the tensor-core kernel)");
  SSB_CHECK(a.w_host && a.Cin > 0 && a.N > 0 && a.k >= 1 && a.dilation >= 1, "op_gemm: bad weight shape");
  SSB_CHECK(!a.gate || a.N % 2 == 0, "op_gemm: the gate packing needs an even N");
  const int64_t reach = (int64_t)(a.k - 1) / 2 * a.dilation;
  SSB_CHECK(reach <= GUARD, "op_gemm: conv reach (k - 1) / 2 * dilation = " + std::to_string(reach) + " exceeds the " +
                                std::to_string(GUARD) + " guard rows between utterances");
  HostTensor wt, bt;
  wt.data = a.w_host; wt.shape = {a.N, a.Cin, a.k};
  bt.data = a.b_host; bt.shape = {a.N};
  const PackMode pm = a.gate ? PACK_GATE_SIG_TANH : PACK_PLAIN;
  if (pack_conv(w->pool, &wt, a.b_host ? &bt : nullptr, a.dilation, pm, &w->cv)) return -1;
  if (a.path == 1) {
    SSB_CHECK(tc_available(), "tensor-core path unavailable (cuTensorMapEncodeTiled)");
    if (pack_conv_tc(w->pool, &wt, a.dilation, pm, w->cv.bias, &w->ct)) return -1;
    SSB_CHECK(w->ct.ok, "op_gemm: shape not eligible for the tensor-core path (Cin % 64, N % 64)");
  }
  return 0;
}

// One conv_gemm / conv_gemm_tc call over the layout s; every epilogue field of a goes to the kernel as it is.
static int op_launch(Ctx& c, const SeqDev& s, const ssb_op_gemm_args& a, const OpWeights& w) {
  if (a.path == 0) {
    ConvGemm g = make_gemm(w.cv, s, a.a, a.lda);
    g.a_act = a.a_act; g.a_slope = a.a_slope; g.a_scale = a.a_scale;
    Epi& e = g.e;
    e.mode = a.mode; e.add = a.add; e.ld_add = a.ld_add; e.alpha = a.alpha; e.act = a.act; e.act_slope = a.act_slope;
    e.res = a.res; e.ld_res = a.ld_res; e.beta = a.beta; e.rowmask = a.rowmask;
    e.out = a.out; e.ldo = a.ldo; e.accum = a.accum; e.gamma = a.gamma;
    e.out2 = a.out2; e.ldo2 = a.ldo2; e.vec2 = a.vec2;
    e.out2_h = (__half*)a.oh; e.out2_l = (__half*)a.ol; e.ldh = a.ldh; e.plane_act = a.plane_act; e.plane_slope = a.plane_slope;
    e.skip = a.skip; e.ld_skip = a.ld_skip; e.C = a.C; e.skip_init = a.skip_init;
    return conv_gemm(c, g);
  }
  GemmTC g = make_gemm_tc(w.ct, s, (const __half*)a.a_hi, (const __half*)a.a_lo);
  g.single_pass = a.single_pass != 0;
  EpiTC& e = g.e;
  e.mode = a.mode; e.out = a.out; e.ldo = a.ldo;
  e.oh = (__half*)a.oh; e.ol = (__half*)a.ol; e.ldh = a.ldh;
  e.add = a.add; e.ld_add = a.ld_add; e.res = a.res; e.ld_res = a.ld_res;
  e.rh = (const __half*)a.rh; e.rl = (const __half*)a.rl; e.ld_rh = a.ld_rh; e.vec1 = a.vec1; e.beta = a.beta;
  e.vec2 = a.vec2; e.skip = a.skip; e.ld_skip = a.ld_skip; e.C = a.C; e.skip_init = a.skip_init;
  e.act = a.act; e.act_slope = a.act_slope; e.accum = a.accum; e.gamma = a.gamma;
  e.plane_act = a.plane_act; e.plane_slope = a.plane_slope; e.alpha = a.alpha; e.rowmask = a.rowmask;
  e.n_valid = a.n_valid; e.skip_tiled = a.skip_tiled; e.out_nb = a.out_nb; e.out_bs = a.out_bs;
  e.sh = (__half*)a.sh; e.sl = (__half*)a.sl;
  return conv_gemm_tc(c, g);
}

// Waits for the call's work, frees its workspace and reports an asynchronous failure.
static int op_finish(void* ws, void* stream, int rc, const char* what) {
  const cudaError_t se = cudaStreamSynchronize((cudaStream_t)stream);
  cudaFree(ws);
  if (rc == 0 && se != cudaSuccess) {
    ssb::set_error(std::string(what) + ": " + cudaGetErrorString(se));
    rc = -2;
  }
  return rc;
}

// ---- one attention call at unit-test granularity (ssb_op_attention_ex) ---------------------------------------------------
// Path 1 first transposes V's planes into V^T scratch taken from c, as the stage drivers do.  Every check of the call
// runs before that transpose, so a refused call launches nothing.
static int op_attn_launch(Ctx& c, const SeqDev& dq, const SeqDev& dk, const ssb_op_attention_args& a) {
  if (a.path == 0) {
    AttnArgs t;
    t.utt_q = dq.utt; t.utt_k = dk.utt; t.B = a.B; t.max_q = dq.maxlen; t.heads = a.heads;
    t.Q = a.q; t.ldq = a.ldq; t.K = a.k; t.ldk = a.ldk; t.V = a.v; t.ldv = a.ldv;
    t.keymask = a.keymask; t.scale = a.scale; t.out = a.out; t.ldo = a.ldo;
    return attention(c, t);
  }
  AttnTCArgs t;
  t.utt_q = dq.utt; t.utt_k = dk.utt; t.B = a.B; t.max_q = dq.maxlen; t.heads = a.heads;
  t.Qh = (const __half*)a.q_hi; t.Ql = (const __half*)a.q_lo; t.rows_q = dq.rows; t.ldq = a.ldq; t.qcol0 = a.qcol0;
  t.Kh = (const __half*)a.k_hi; t.Kl = (const __half*)a.k_lo; t.rows_k = dk.rows; t.ldk = a.ldk; t.kcol0 = a.kcol0;
  t.ldvt = (dk.rows + 7) & ~int64_t(7);
  t.keymask = a.keymask; t.scale = a.scale;
  t.out = a.out; t.ldo = a.ldo; t.oh = (__half*)a.oh; t.ol = (__half*)a.ol; t.ldh = a.ldh;
  if (attention_tc_check(t)) return -1;  // before the V^T scratch exists; it comes from c, 256-byte aligned
  const int w = a.heads * 128;
  SSB_CHECK(a.ldv % 8 == 0 && a.vcol0 >= 0 && a.vcol0 % 8 == 0 && a.vcol0 + w <= a.ldv,
            "op_attention: V's ldv and vcol0 must be multiples of 8 and vcol0 + heads x 128 must not exceed ldv");
  __half* vth = c.alloc<__half>((size_t)t.ldvt * w);
  __half* vtl = c.alloc<__half>((size_t)t.ldvt * w);
  SSB_CHECK(!c.failed, "op_attention: workspace too small");
  t.Vth = vth; t.Vtl = vtl;
  if (transpose_planes(c, (const __half*)a.v_hi, (const __half*)a.v_lo, a.ldv, a.vcol0, dk.rows, w, vth, vtl, t.ldvt)) return -1;
  return attention_tc(c, t);
}

extern "C" {

int ssb_version(void) { return 104; }
const char* ssb_last_error(void) { return ssb::last_error(); }

int ssb_model_create(ssb_model_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_hparams* hp) {
  return ssb_model_create_ex(out, tensors, n, hp, SSB_MEL_DECODER_DIFFSINGER);
}
int ssb_model_create_ex(ssb_model_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_hparams* hp,
                        int32_t mel_decoder) {
  return ssb_model_create_ex2(out, tensors, n, hp, mel_decoder, SSB_F0_GEN_GMDIFF);
}
int ssb_model_create_ex2(ssb_model_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_hparams* hp,
                         int32_t mel_decoder, int32_t f0_gen) {
  const ssb_model_switches all_on = {1, 1, 1, 1};
  return ssb_model_create_ex3(out, tensors, n, hp, mel_decoder, f0_gen, &all_on);
}
int ssb_model_create_ex3(ssb_model_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_hparams* hp,
                         int32_t mel_decoder, int32_t f0_gen, const ssb_model_switches* sw) {
  return ssb_model_create_ex4(out, tensors, n, hp, mel_decoder, f0_gen, sw, 0);
}
int ssb_model_create_ex4(ssb_model_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_hparams* hp,
                         int32_t mel_decoder, int32_t f0_gen, const ssb_model_switches* sw, int32_t use_spk_id) {
  if (out) *out = nullptr;
  SSB_CHECK(mel_decoder == SSB_MEL_DECODER_DIFFSINGER || mel_decoder == SSB_MEL_DECODER_PRODIFF ||
                mel_decoder == SSB_MEL_DECODER_FFT,
            "ssb_model_create_ex: unknown mel_decoder " + std::to_string(mel_decoder) +
                " (SSB_MEL_DECODER_DIFFSINGER = 0, SSB_MEL_DECODER_PRODIFF = 1, SSB_MEL_DECODER_FFT = 2)");
  SSB_CHECK(f0_gen == SSB_F0_GEN_GMDIFF || f0_gen == SSB_F0_GEN_CONV,
            "ssb_model_create_ex2: unknown f0_gen " + std::to_string(f0_gen) +
                " (SSB_F0_GEN_GMDIFF = 0, SSB_F0_GEN_CONV = 1)");
  SSB_CHECK(sw, "ssb_model_create_ex3: null switches");
  SSB_CHECK(use_spk_id == 0 || use_spk_id == 1,
            "ssb_model_create_ex4: use_spk_id must be 0 or 1, got " + std::to_string(use_spk_id));
  {
    const char* names[4] = {"emo", "style", "umln", "use_txt_cond"};
    const int32_t vals[4] = {sw->emo, sw->style, sw->umln, sw->use_txt_cond};
    for (int i = 0; i < 4; ++i)
      SSB_CHECK(vals[i] == 0 || vals[i] == 1, std::string("ssb_model_create_ex3: switch ") + names[i] + " must be 0 or 1, got " +
                                                  std::to_string(vals[i]));
  }
  SSB_CHECK(out && tensors && hp, "ssb_model_create: null argument");
  TensorMap tm;
  if (to_map(tensors, n, &tm)) return -1;
  if (mel_decoder == SSB_MEL_DECODER_DIFFSINGER) {  // ln_proj = Linear(cond_hs, H), cond_hs of stylesinger.py:92-100
    const auto it = tm.t.find("ln_proj.weight");
    if (it != tm.t.end()) {
      const std::vector<int64_t>& sh = it->second.shape;
      const int w = cond_width(*sw);
      SSB_CHECK(sh.size() == 2 && sh[0] == hp->hidden_size && sh[1] == w,
                "ssb_model_create_ex3: ln_proj.weight must be [" + std::to_string(hp->hidden_size) + ", " + std::to_string(w) +
                    "] = 80 + 256 x (1 + use_txt_cond " + std::to_string(sw->use_txt_cond) + " + emo " +
                    std::to_string(sw->emo) + " + style " + std::to_string(sw->style) + "), got [" +
                    (sh.empty() ? std::string() : std::to_string(sh[0])) + (sh.size() > 1 ? ", " + std::to_string(sh[1]) : "") +
                    (sh.size() > 2 ? ", ..." : "") + "]");
    }
  }
  ssb_model* m = new ssb_model();
  if (build_model(tm, *hp, &m->m, mel_decoder, f0_gen, *sw, use_spk_id != 0) != 0) {
    delete m;
    return -1;
  }
  *out = m;
  return 0;
}
void ssb_model_free(ssb_model_t* m) {
  if (!m) return;
  if (m->m.aux_stream) {
    cudaStreamSynchronize(m->m.aux_stream);
    cudaEventDestroy(m->m.ev_fork);
    cudaEventDestroy(m->m.ev_join);
    cudaStreamDestroy(m->m.aux_stream);
  }
  delete m;
}

int ssb_model_set_schedule(ssb_model_t* m, int32_t which, int32_t T, const float* step_emb, const float* gauss_tab,
                           const float* multi_tab, void* stream) {
  SSB_CHECK(m, "null model");
  return set_schedule(&m->m, which, T, step_emb, gauss_tab, multi_tab, (cudaStream_t)stream);
}

int ssb_model_set_mel_k_step(ssb_model_t* m, int32_t K) {
  SSB_CHECK(m, "null model");
  SSB_CHECK(m->m.mel_decoder != SSB_MEL_DECODER_FFT,
            "ssb_model_set_mel_k_step: a model with the FFT mel decoder (SSB_MEL_DECODER_FFT) has no mel sampler and no K_step");
  SSB_CHECK(K >= 0, "ssb_model_set_mel_k_step: K must be >= 0 (0 follows the schedule's T), got " + std::to_string(K));
  SSB_CHECK(m->m.mel_decoder == SSB_MEL_DECODER_DIFFSINGER,
            "ssb_model_set_mel_k_step: a ProDiff model has no K_step (ProDiffusion.forward never reads it)");
  m->m.mel_k_step = K;
  return 0;
}

size_t ssb_durations_workspace_bytes(const ssb_model_t* m, const ssb_acoustic_inputs* in) {
  Ctx c = make_ctx(nullptr, 0, nullptr, true);
  ssb_acoustic_outputs o;
  memset(&o, 0, sizeof(o));
  if (run_acoustic(c, m->m, *in, o, true, nullptr, nullptr) != 0) return 0;
  return c.high + 4096;
}
int ssb_predict_durations(const ssb_model_t* m, const ssb_acoustic_inputs* in, int32_t* dur_out, float* logdur_out,
                          void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && in && workspace, "null argument");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  ssb_acoustic_outputs o;
  memset(&o, 0, sizeof(o));
  return run_acoustic(c, m->m, *in, o, true, dur_out, logdur_out);
}
size_t ssb_acoustic_workspace_bytes(const ssb_model_t* m, const ssb_acoustic_inputs* in) {
  Ctx c = make_ctx(nullptr, 0, nullptr, true);
  ssb_acoustic_outputs o;
  memset(&o, 0, sizeof(o));
  o.mel_out = (float*)(uintptr_t)256;
  if (run_acoustic(c, m->m, *in, o, false, nullptr, nullptr) != 0) return 0;
  return c.high + 4096;
}
int ssb_acoustic_forward(const ssb_model_t* m, const ssb_acoustic_inputs* in, const ssb_acoustic_outputs* out,
                         void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && in && out && workspace, "null argument");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  return run_acoustic(c, m->m, *in, *out, false, nullptr, nullptr);
}
int ssb_acoustic_forward_keyed(const ssb_model_t* m, const ssb_acoustic_inputs* in, const uint64_t* utt_seeds,
                               const ssb_acoustic_outputs* out, void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && in && out && workspace, "null argument");
  SSB_CHECK(utt_seeds, "ssb_acoustic_forward_keyed: utt_seeds (one seed per utterance) is required");
  SSB_CHECK(!in->mel_noise && !in->f0_gauss_noise[0] && !in->f0_gauss_noise[1] && !in->f0_unif_noise[0] &&
                !in->f0_unif_noise[1],
            "ssb_acoustic_forward_keyed: per-utterance seeds key the in-kernel noise; injected noise must be NULL");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  return run_acoustic(c, m->m, *in, *out, false, nullptr, nullptr, utt_seeds);
}

// The standalone mel-sampler entries need a mel DiffNet, which an FFT model does not have
static int need_mel_diffnet(const Model& m, const char* what) {
  SSB_CHECK(m.mel_decoder != SSB_MEL_DECODER_FFT,
            std::string(what) + ": a model with the FFT mel decoder (SSB_MEL_DECODER_FFT) has no mel DiffNet");
  return 0;
}

static int mel_diff_impl(Ctx& c, const Model& m, const float* cond, const float* coarse, const int32_t* offs, int B,
                         const float* noise, uint64_t seed, float* mel_out) {
  RUN(need_mel_diffnet(m, "ssb_mel_diffusion_sample"));
  SSB_CHECK(m.mel_decoder == SSB_MEL_DECODER_DIFFSINGER,
            "ssb_mel_diffusion_sample: the DDPM sampler needs a DiffSinger model; use ssb_mel_prodiff_sample on a ProDiff model");
  Seq q;
  q.build(offs, B);
  q.seed = seed;
  SeqDev s;
  RUN(upload_layout(c, q, 1, &s));
  float* cg = alloc_rows(c, s, 256);
  float* co = alloc_rows(c, s, 80);
  WS_OK(c);
  RUN(pack_rows(c, s, cond, 256, cg, 256, 256));
  RUN(pack_rows(c, s, coarse, 80, co, 80, 80));
  return run_mel_diffusion(c, m, s, cg, co, noise, mel_out, &q);
}
static int mel_plms_impl(Ctx& c, const Model& m, const float* cond, const float* coarse, const int32_t* offs, int B,
                         const float* q_noise, uint64_t seed, int interval, float* mel_out) {
  RUN(need_mel_diffnet(m, "ssb_mel_diffusion_sample_plms"));
  Seq q;
  q.build(offs, B);
  q.seed = seed;
  SeqDev s;
  RUN(upload_layout(c, q, 1, &s));
  float* cg = alloc_rows(c, s, 256);
  float* co = alloc_rows(c, s, 80);
  WS_OK(c);
  RUN(pack_rows(c, s, cond, 256, cg, 256, 256));
  RUN(pack_rows(c, s, coarse, 80, co, 80, 80));
  return run_mel_diffusion_plms(c, m, s, cg, co, q_noise, interval, mel_out);
}
static int mel_prodiff_impl(Ctx& c, const Model& m, const float* cond, const int32_t* offs, int B, const float* noise,
                            uint64_t seed, float* mel_out) {
  RUN(need_mel_diffnet(m, "ssb_mel_prodiff_sample"));
  SSB_CHECK(m.mel_decoder == SSB_MEL_DECODER_PRODIFF,
            "ssb_mel_prodiff_sample: the ProDiff sampler needs a model created with SSB_MEL_DECODER_PRODIFF");
  Seq q;
  q.build(offs, B);
  q.seed = seed;
  SeqDev s;
  RUN(upload_layout(c, q, 1, &s));
  float* cg = alloc_rows(c, s, 256);
  WS_OK(c);
  RUN(pack_rows(c, s, cond, 256, cg, 256, 256));
  return run_mel_diffusion(c, m, s, cg, nullptr, noise, mel_out, &q);
}
size_t ssb_mel_prodiff_workspace_bytes(const ssb_model_t* m, const int32_t* frame_offsets, int32_t B) {
  Ctx c = make_ctx(nullptr, 0, nullptr, true);
  if (mel_prodiff_impl(c, m->m, nullptr, frame_offsets, B, nullptr, 0, nullptr) != 0) return 0;
  return c.high + 4096;
}
int ssb_mel_prodiff_sample(const ssb_model_t* m, const float* cond, const int32_t* frame_offsets, int32_t B,
                           const float* noise, uint64_t seed, float* mel_out, void* workspace, size_t workspace_bytes,
                           void* stream) {
  SSB_CHECK(m && cond && frame_offsets && mel_out && workspace, "null argument");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  return mel_prodiff_impl(c, m->m, cond, frame_offsets, B, noise, seed, mel_out);
}
size_t ssb_mel_diffusion_plms_workspace_bytes(const ssb_model_t* m, const int32_t* frame_offsets, int32_t B) {
  Ctx c = make_ctx(nullptr, 0, nullptr, true);
  if (mel_plms_impl(c, m->m, nullptr, nullptr, frame_offsets, B, nullptr, 0, 1, nullptr) != 0) return 0;
  return c.high + 4096;
}
int ssb_mel_diffusion_sample_plms(const ssb_model_t* m, const float* cond, const float* coarse_mel,
                                  const int32_t* frame_offsets, int32_t B, const float* q_noise, uint64_t seed,
                                  int32_t interval, float* mel_out, void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && cond && coarse_mel && frame_offsets && mel_out && workspace, "null argument");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  return mel_plms_impl(c, m->m, cond, coarse_mel, frame_offsets, B, q_noise, seed, interval, mel_out);
}
size_t ssb_mel_diffusion_workspace_bytes(const ssb_model_t* m, const int32_t* frame_offsets, int32_t B) {
  Ctx c = make_ctx(nullptr, 0, nullptr, true);
  if (mel_diff_impl(c, m->m, nullptr, nullptr, frame_offsets, B, nullptr, 0, nullptr) != 0) return 0;
  return c.high + 4096;
}
int ssb_mel_diffusion_sample(const ssb_model_t* m, const float* cond, const float* coarse_mel,
                             const int32_t* frame_offsets, int32_t B, const float* noise, uint64_t seed,
                             float* mel_out, void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && cond && coarse_mel && frame_offsets && mel_out && workspace, "null argument");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  return mel_diff_impl(c, m->m, cond, coarse_mel, frame_offsets, B, noise, seed, mel_out);
}

int ssb_denoiser_eval(const ssb_model_t* m, int32_t which, const float* x, const int32_t* uv, int32_t t,
                      const float* cond, const int32_t* frame_offsets, int32_t B, float* out, void* workspace,
                      size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && x && cond && frame_offsets && out && workspace && which >= 0 && which <= 2, "bad argument");
  SSB_CHECK(which == 0 || m->m.f0_gen == SSB_F0_GEN_GMDIFF,
            "ssb_denoiser_eval: a model with the conv F0 generator (SSB_F0_GEN_CONV) has no F0 denoisers (which = 1 / 2)");
  if (which == 0) RUN(need_mel_diffnet(m->m, "ssb_denoiser_eval(which = 0)"));
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  Seq q;
  q.build(frame_offsets, B);
  SeqDev s;
  RUN(upload_layout(c, q, 1, &s));
  return denoiser_eval_api(c, m->m, which, s, x, uv, t, cond, out);
}

int ssb_f0_diffusion_sample(const ssb_model_t* m, int32_t which, const float* cond, const float* clip_lo,
                            const float* clip_hi, const int32_t* frame_offsets, int32_t B, const float* gauss_noise,
                            const float* unif_noise, uint64_t seed, float* f0_norm_out, int32_t* uv_out,
                            void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && cond && clip_lo && clip_hi && frame_offsets && f0_norm_out && uv_out && workspace, "null argument");
  SSB_CHECK(which == 0 || which == 1, "which must be 0 or 1");
  SSB_CHECK(m->m.f0_gen == SSB_F0_GEN_GMDIFF,
            "ssb_f0_diffusion_sample: a model with the conv F0 generator (SSB_F0_GEN_CONV) has no F0 sampler; use "
            "ssb_pitch_predictor");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  Seq q;
  q.build(frame_offsets, B);
  q.seed = seed;
  SeqDev s;
  RUN(upload_layout(c, q, 1, &s));
  float* cg = alloc_rows(c, s, 256);
  float* lo = alloc_rows(c, s, 1);
  float* hi = alloc_rows(c, s, 1);
  float* z = alloc_rows(c, s, 1);
  int32_t* uv = alloc_rows_i32(c, s);
  WS_OK(c);
  RUN(pack_rows(c, s, cond, 256, cg, 256, 256));
  RUN(pack_rows(c, s, clip_lo, 1, lo, 1, 1));
  RUN(pack_rows(c, s, clip_hi, 1, hi, 1, 1));
  RUN(run_f0_diffusion(c, m->m, which, s, cg, lo, hi, gauss_noise, unif_noise, z, uv));
  RUN(unpack_rows(c, s, z, 1, f0_norm_out, 1, 1));
  RUN(unpack_rows_i32(c, s, uv, uv_out));
  return 0;
}

static int pitch_predictor_impl(Ctx& c, const Model& m, int which, const float* x, const int32_t* offs, int B, float* out) {
  SSB_CHECK(m.f0_gen == SSB_F0_GEN_CONV,
            "ssb_pitch_predictor: the PitchPredictors need a model created with SSB_F0_GEN_CONV (a gmdiff model samples F0)");
  Seq q;
  q.build(offs, B);
  SSB_CHECK(q.maxlen + 2 <= m.pos_rows, "frame sequence longer than __pos_table");
  SeqDev s;
  RUN(upload_layout(c, q, 1, &s));
  float* xg = alloc_rows(c, s, 256);
  float* og = alloc_rows(c, s, 2);
  WS_OK(c);
  RUN(pack_rows(c, s, x, 256, xg, 256, 256));
  RUN(run_pitch_predictor(c, m, which, s, xg, og, long_batch_tc(m, s)));
  return unpack_rows(c, s, og, 2, out, 2, 2);
}
size_t ssb_pitch_predictor_workspace_bytes(const ssb_model_t* m, const int32_t* frame_offsets, int32_t B) {
  Ctx c = make_ctx(nullptr, 0, nullptr, true);
  if (pitch_predictor_impl(c, m->m, 0, nullptr, frame_offsets, B, nullptr) != 0) return 0;
  return c.high + 4096;
}
int ssb_pitch_predictor(const ssb_model_t* m, int32_t which, const float* x, const int32_t* frame_offsets, int32_t B,
                        float* out, void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && x && frame_offsets && out && workspace, "null argument");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  return pitch_predictor_impl(c, m->m, which, x, frame_offsets, B, out);
}

// ---- per-registry drop-ins (FS_ENCODERS / FS_DECODERS 'fft', StyleSinger.get_style) ------------------------------------
static int fft_encoder_impl(Ctx& c, const Model& m, const int32_t* tokens, const int32_t* offs, int B, float* out) {
  Seq q;
  q.build(offs, B);
  SSB_CHECK(q.maxlen + 2 <= m.pos_rows, "sequence longer than __pos_table");
  SeqDev sp;
  RUN(upload_layout(c, q, 1, &sp));
  int32_t* tok = alloc_rows_i32(c, sp);
  float* srcmask = alloc_rows(c, sp, 1);
  float* enc = alloc_rows(c, sp, 256);
  WS_OK(c);
  RUN(pack_rows_i32(c, sp, tokens, tok));
  RUN(run_encoder(c, m, sp, tok, nullptr, nullptr, nullptr, srcmask, enc));
  return unpack_rows(c, sp, enc, 256, out, 256, 256);
}
static int fft_decoder_impl(Ctx& c, const Model& m, const float* x, const int32_t* offs, int B, float* out) {
  Seq q;
  q.build(offs, B);
  SSB_CHECK(q.maxlen + 2 <= m.pos_rows, "frame sequence longer than __pos_table");
  SeqDev sf;
  RUN(upload_layout(c, q, 1, &sf));
  float* xin = alloc_rows(c, sf, 256);
  float* xd = alloc_rows(c, sf, 256);
  WS_OK(c);
  RUN(pack_rows(c, sf, x, 256, xin, 256, 256));
  RUN(run_fft_decoder(c, m, sf, xin, xd, long_batch_tc(m, sf)));
  return unpack_rows(c, sf, xd, 256, out, 256, 256);
}
static int get_style_impl(Ctx& c, const Model& m, const float* dec_inp, const int32_t* foffs, const float* ref_mels,
                          const float* ref_f0, const int32_t* roffs, int B, float* style_out, int32_t* codes_out) {
  SSB_CHECK(m.sw.style, "ssb_get_style: a model without style (switch style = 0) has no style adaptor");
  Seq qf, qr;
  qf.build(foffs, B);
  qr.build(roffs, B);
  SSB_CHECK(qf.maxlen + 2 <= m.pos_rows && qr.maxlen + 2 <= m.pos_rows, "sequence longer than __pos_table");
  SeqDev sf, sr;
  RUN(upload_layout(c, qf, 1, &sf));
  RUN(upload_layout(c, qr, 1, &sr));
  float* dec0 = alloc_rows(c, sf, 256);
  float* style = alloc_rows(c, sf, 256);
  float* ref = alloc_rows(c, sr, 80);
  float* reff0 = alloc_rows(c, sr, 1);
  int32_t* codes = alloc_rows_i32(c, sr, m.hp.rq_depth);
  WS_OK(c);
  RUN(pack_rows(c, sf, dec_inp, 256, dec0, 256, 256));
  RUN(pack_rows(c, sr, ref_mels, 80, ref, 80, 80));
  RUN(pack_rows(c, sr, ref_f0, 1, reff0, 1, 1));
  RUN(run_style(c, m, sf, sr, dec0, ref, reff0, style, codes, nullptr));
  RUN(unpack_rows(c, sf, style, 256, style_out, 256, 256));
  if (codes_out)
    for (int d = 0; d < m.hp.rq_depth; ++d) RUN(unpack_cols_i32(c, sr, codes, m.hp.rq_depth, d, codes_out));
  return 0;
}

size_t ssb_fft_workspace_bytes(const ssb_model_t* m, int32_t which, const int32_t* offsets, int32_t B) {
  Ctx c = make_ctx(nullptr, 0, nullptr, true);
  const int rc = which == 0 ? fft_encoder_impl(c, m->m, nullptr, offsets, B, nullptr)
                            : fft_decoder_impl(c, m->m, nullptr, offsets, B, nullptr);
  return rc == 0 ? c.high + 4096 : 0;
}
int ssb_fft_encoder(const ssb_model_t* m, const int32_t* txt_tokens, const int32_t* ph_offsets, int32_t B, float* out,
                    void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && txt_tokens && ph_offsets && out && workspace, "null argument");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  return fft_encoder_impl(c, m->m, txt_tokens, ph_offsets, B, out);
}
int ssb_fft_decoder(const ssb_model_t* m, const float* x, const int32_t* frame_offsets, int32_t B, float* out,
                    void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && x && frame_offsets && out && workspace, "null argument");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  return fft_decoder_impl(c, m->m, x, frame_offsets, B, out);
}
size_t ssb_get_style_workspace_bytes(const ssb_model_t* m, const int32_t* frame_offsets, const int32_t* ref_offsets, int32_t B) {
  Ctx c = make_ctx(nullptr, 0, nullptr, true);
  return get_style_impl(c, m->m, nullptr, frame_offsets, nullptr, nullptr, ref_offsets, B, nullptr, nullptr) == 0 ? c.high + 4096 : 0;
}
int ssb_get_style(const ssb_model_t* m, const float* decoder_inp, const int32_t* frame_offsets, const float* ref_mels,
                  const float* ref_f0, const int32_t* ref_offsets, int32_t B, float* style_out, int32_t* codes_out,
                  void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && decoder_inp && frame_offsets && ref_mels && ref_f0 && ref_offsets && style_out && workspace, "null argument");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  return get_style_impl(c, m->m, decoder_inp, frame_offsets, ref_mels, ref_f0, ref_offsets, B, style_out, codes_out);
}

int ssb_rvq_lookup(const ssb_model_t* m, const float* x, const int32_t* ref_offsets, int32_t B, float* quant_out,
                   int32_t* codes_out, void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && x && ref_offsets && quant_out && codes_out && workspace, "null argument");
  SSB_CHECK(m->m.sw.style, "ssb_rvq_lookup: a model without style (switch style = 0) has no RVQ codebooks");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  Seq q;
  q.build(ref_offsets, B);
  SeqDev s;
  RUN(upload_layout(c, q, 1, &s));
  const int D = m->m.hp.rq_depth;
  float* xg = alloc_rows(c, s, 256);
  float* zq = alloc_rows(c, s, 256);
  int32_t* codes = alloc_rows_i32(c, s, D);
  WS_OK(c);
  RUN(pack_rows(c, s, x, 256, xg, 256, 256));
  RUN(rvq_lookup(c, s, xg, 256, m->m.codebooks, m->m.cb_norm2, m->m.hp.n_rq, D, zq, 256, codes));
  RUN(unpack_rows(c, s, zq, 256, quant_out, 256, 256));
  for (int d = 0; d < D; ++d) RUN(unpack_cols_i32(c, s, codes, D, d, codes_out));
  return 0;
}

int ssb_vocoder_create(ssb_vocoder_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_vocoder_config* cfg) {
  SSB_CHECK(out && tensors && cfg, "ssb_vocoder_create: null argument");
  ssb_vocoder_config_ex ex;
  memset(&ex, 0, sizeof(ex));
  ex.n_up = cfg->n_up;
  memcpy(ex.up_rates, cfg->up_rates, sizeof(ex.up_rates));
  memcpy(ex.up_kernels, cfg->up_kernels, sizeof(ex.up_kernels));
  ex.initial_channel = cfg->initial_channel;
  ex.n_res = cfg->n_res;
  memcpy(ex.res_kernels, cfg->res_kernels, sizeof(ex.res_kernels));
  memcpy(ex.res_dilations, cfg->res_dilations, sizeof(ex.res_dilations));
  ex.use_pitch_embed = cfg->use_pitch_embed;
  ex.sample_rate = cfg->sample_rate;
  ex.resblock = 1;
  return ssb_vocoder_create_ex(out, tensors, n, &ex);
}

// The layout rules of ssb_vocoder_create_ex, checked on the config alone (before any allocation)
static int check_vocoder_config(const ssb_vocoder_config_ex& cfg) {
  const std::string w = "ssb_vocoder_create: ";
  SSB_CHECK(cfg.resblock == 1 || cfg.resblock == 2,
            w + "resblock must be 1 (ResBlock1) or 2 (ResBlock2), got " + std::to_string(cfg.resblock));
  SSB_CHECK(cfg.n_up >= 1 && cfg.n_up <= 8 && cfg.n_res >= 1 && cfg.n_res <= 4, w + "vocoder: unsupported config");
  const int nd = cfg.resblock == 1 ? 3 : 2;  // ResBlock1 reads dilation[0..2], ResBlock2 dilation[0..1]
  for (int j = 0; j < cfg.n_res; ++j)
    for (int m = 0; m < nd; ++m)
      SSB_CHECK(cfg.res_dilations[j][m] >= 1, w + "dilation " + std::to_string(cfg.res_dilations[j][m]) + " of resblock " +
                                                  std::to_string(j) + " (entry " + std::to_string(m) + ") is below 1");
  int rate = 1;
  for (int i = 0; i < cfg.n_up; ++i) {
    SSB_CHECK(cfg.up_rates[i] >= 1, w + "upsample rate " + std::to_string(i) + " is below 1");
    rate *= cfg.up_rates[i];
    const int div = 2 << i;
    const int C = cfg.initial_channel / div;
    SSB_CHECK(cfg.initial_channel > 0 && cfg.initial_channel % div == 0 && (C % 32 == 0 || C == 16 || C == 8),
              w + "stage " + std::to_string(i) + " has initial_channel / 2^" + std::to_string(i + 1) + " = " +
                  std::to_string(cfg.initial_channel) + " / " + std::to_string(div) +
                  " channels: it must be a multiple of 32, or 16 or 8");
    if (C < 32)
      SSB_CHECK(rate % (64 / C) == 0, w + "stage " + std::to_string(i) + " has " + std::to_string(C) +
                                          " channels and cumulative upsampling rate " + std::to_string(rate) +
                                          ", which is not a multiple of 64 / " + std::to_string(C) +
                                          " (its ResBlock convs run over groups of that many samples)");
  }
  return 0;
}

int ssb_vocoder_create_ex(ssb_vocoder_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_vocoder_config_ex* cfg) {
  SSB_CHECK(out, "ssb_vocoder_create: null argument");
  *out = nullptr;
  SSB_CHECK(tensors && cfg, "ssb_vocoder_create: null argument");
  if (check_vocoder_config(*cfg)) return -1;
  TensorMap tm;
  if (to_map(tensors, n, &tm)) return -1;
  ssb_vocoder* v = new ssb_vocoder();
  if (build_vocoder(tm, *cfg, &v->v) != 0) {
    delete v;
    return -1;
  }
  *out = v;
  return 0;
}
void ssb_vocoder_free(ssb_vocoder_t* v) { delete v; }

size_t ssb_vocoder_workspace_bytes(const ssb_vocoder_t* v, const int32_t* frame_offsets, int32_t B) {
  Ctx c = make_ctx(nullptr, 0, nullptr, true);
  Seq q;
  q.build(frame_offsets, B);
  if (run_vocoder(c, v->v, q, nullptr, (const float*)(uintptr_t)256, nullptr, nullptr, nullptr) != 0) return 0;
  return c.high + 4096;
}
int ssb_hifigan_generate(const ssb_vocoder_t* v, const float* mel, const float* f0, const int32_t* frame_offsets,
                         int32_t B, const float* rand_ini, const float* src_noise, uint64_t seed, float* wav_out,
                         void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(v && mel && frame_offsets && wav_out && workspace, "null argument");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  Seq q;
  q.build(frame_offsets, B);
  q.seed = seed;
  return run_vocoder(c, v->v, q, mel, f0, rand_ini, src_noise, wav_out);
}
int ssb_hifigan_generate_keyed(const ssb_vocoder_t* v, const float* mel, const float* f0, const int32_t* frame_offsets,
                               int32_t B, const uint64_t* utt_seeds, float* wav_out, void* workspace,
                               size_t workspace_bytes, void* stream) {
  SSB_CHECK(v && mel && frame_offsets && wav_out && workspace, "null argument");
  SSB_CHECK(utt_seeds, "ssb_hifigan_generate_keyed: utt_seeds (one seed per utterance) is required");
  Ctx c = make_ctx(workspace, workspace_bytes, stream);
  Seq q;
  q.build(frame_offsets, B);
  q.utt_seeds = utt_seeds;
  return run_vocoder(c, v->v, q, mel, f0, nullptr, nullptr, wav_out);
}

int ssb_model_set_tensor_cores(ssb_model_t* m, int32_t enable) {
  SSB_CHECK(m, "null model");
  m->m.use_tc = enable != 0 && tc_available();
  return m->m.use_tc ? 1 : 0;
}

int ssb_vocoder_set_tensor_cores(ssb_vocoder_t* v, int32_t enable) {
  SSB_CHECK(v, "null vocoder");
  v->v.use_tc = enable != 0 && tc_available();
  return v->v.use_tc ? 1 : 0;
}

int ssb_model_set_mel_precision(ssb_model_t* m, int32_t mode) {
  SSB_CHECK(m, "null model");
  SSB_CHECK(mode == SSB_TC_SPLIT || mode == SSB_TC_FP16,
            "ssb_model_set_mel_precision: mode must be SSB_TC_SPLIT (0) or SSB_TC_FP16 (1), got " + std::to_string(mode));
  m->m.mel_fp16 = mode == SSB_TC_FP16;
  return 0;
}

int ssb_vocoder_set_precision(ssb_vocoder_t* v, int32_t mode) {
  SSB_CHECK(v, "null vocoder");
  SSB_CHECK(mode == SSB_TC_SPLIT || mode == SSB_TC_FP16,
            "ssb_vocoder_set_precision: mode must be SSB_TC_SPLIT (0) or SSB_TC_FP16 (1), got " + std::to_string(mode));
  v->v.fp16 = mode == SSB_TC_FP16;
  return 0;
}

int ssb_model_set_fft_tensor_cores(ssb_model_t* m, int32_t enable) {
  SSB_CHECK(m, "null model");
  m->m.fft_tc = enable != 0;
  return m->m.fft_tc ? 1 : 0;
}

int ssb_model_set_persistent(ssb_model_t* m, int32_t enable) {
  SSB_CHECK(m, "null model");
  m->m.persistent = enable != 0;
  return m->m.persistent ? 1 : 0;
}

int ssb_model_set_persistent_groups(ssb_model_t* m, int32_t enable) {
  SSB_CHECK(m, "null model");
  m->m.persistent_groups = enable != 0;
  return m->m.persistent_groups ? 1 : 0;
}

int ssb_mel_postprocess(float* mel, int64_t n_frames, float vmin, float vmax, int32_t* nonzero_frames, void* stream) {
  SSB_CHECK(mel && nonzero_frames && n_frames >= 0, "bad argument");
  return mel_postprocess_flat((cudaStream_t)stream, mel, n_frames, vmin, vmax, nonzero_frames);
}
int64_t ssb_launch_count(void) { return (int64_t)ssb::g_launches.load(); }
int32_t ssb_set_attention_tensor_cores(int32_t enable) { return ssb::set_attention_tc_enabled(enable); }
int64_t ssb_attention_launch_count(int32_t tc) { return tc == 0 || tc == 1 ? (int64_t)ssb::g_attn_launches[tc].load() : 0; }
int64_t ssb_variant_launch_count(const char* variant) { return variant ? (int64_t)ssb::variant_launch_count(variant) : 0; }
int32_t ssb_variant_names(char* buf, int32_t cap) { return buf && cap > 0 ? ssb::variant_names(buf, cap) : 0; }
void ssb_tensor_map_cache_stats(int64_t* encodes, int64_t* hits) {
  long long e = 0, h = 0;
  ssb::tensor_map_cache_stats(&e, &h);
  if (encodes) *encodes = e;
  if (hits) *hits = h;
}

int ssb_op_gemm(const ssb_op_gemm_args* a, void* stream) {
  SSB_CHECK(a && a->frame_offsets && a->B >= 1, "ssb_op_gemm: null argument");
  OpWeights w;
  if (op_pack(*a, &w)) return -1;
  SSB_CHECK(a->path == 1 ? (a->a_hi && (a->a_lo || a->single_pass)) : a->a != nullptr, "ssb_op_gemm: no A operand");
  Seq q;
  q.build(a->frame_offsets, a->B);
  SSB_CHECK(a->rows == q.rows(), "ssb_op_gemm: rows is " + std::to_string(a->rows) + ", the layout has " +
                                     std::to_string(q.rows()));
  const size_t bytes = ((size_t)q.ntiles() + (size_t)a->B + 2) * 48 + 4096;  // the layout tables only
  void* ws = nullptr;
  SSB_CUDA(cudaMalloc(&ws, bytes));
  Ctx c = make_ctx(ws, bytes, stream);
  SeqDev s;
  int rc = upload_layout(c, q, 1, &s);
  if (rc == 0) rc = op_launch(c, s, *a, w);
  return op_finish(ws, stream, rc, "ssb_op_gemm");
}

int ssb_op_attention_ex(const ssb_op_attention_args* a, void* stream) {
  SSB_CHECK(a && a->q_offsets && a->k_offsets && a->B >= 1, "ssb_op_attention_ex: null argument");
  SSB_CHECK(a->path == 0 || a->path == 1, "ssb_op_attention_ex: path must be 0 (fp32 kernel) or 1 (wgmma kernel)");
  SSB_CHECK(a->B <= 65535, "ssb_op_attention_ex: B = " + std::to_string(a->B) + " exceeds gridDim.z (65535)");
  if (a->path == 0) {
    SSB_CHECK(a->q && a->k && a->v, "ssb_op_attention_ex: path 0 needs fp32 q, k and v");
    SSB_CHECK(a->out && !a->oh && !a->ol, "ssb_op_attention_ex: path 0 writes fp32 out only (no planes)");
    SSB_CHECK(a->qcol0 == 0 && a->kcol0 == 0 && a->vcol0 == 0,
              "ssb_op_attention_ex: path 0 takes column windows as pointer offsets (qcol0 / kcol0 / vcol0 must be 0)");
  } else {
    SSB_CHECK(tc_available(), "tensor-core path unavailable (cuTensorMapEncodeTiled)");
    SSB_CHECK(a->q_hi && a->q_lo && a->k_hi && a->k_lo && a->v_hi && a->v_lo, "ssb_op_attention_ex: path 1 needs q, k and v planes");
    SSB_CHECK(a->out || (a->oh && a->ol), "ssb_op_attention_ex: no output");
  }
  Seq sq, sk;
  sq.build(a->q_offsets, a->B);
  sk.build(a->k_offsets, a->B);
  SSB_CHECK(a->rows_q == sq.rows(), "ssb_op_attention_ex: rows_q is " + std::to_string(a->rows_q) + ", the query layout has " +
                                        std::to_string(sq.rows()));
  SSB_CHECK(a->rows_k == sk.rows(), "ssb_op_attention_ex: rows_k is " + std::to_string(a->rows_k) + ", the key layout has " +
                                        std::to_string(sk.rows()));
  const int64_t ldvt = (sk.rows() + 7) & ~int64_t(7);
  // the layout tables, and on path 1 the V^T scratch (2 planes of at most 256 x ldvt halves)
  const size_t bytes = ((size_t)sq.ntiles() + (size_t)sk.ntiles() + 2 * (size_t)a->B + 4) * 48 + 4096 +
                       (a->path == 1 ? (size_t)ldvt * 256 * 2 * sizeof(__half) + 512 : 0);
  void* ws = nullptr;
  SSB_CUDA(cudaMalloc(&ws, bytes));
  Ctx c = make_ctx(ws, bytes, stream);
  SeqDev dq, dk;
  int rc = upload_layout(c, sq, 1, &dq);
  if (rc == 0) rc = upload_layout(c, sk, 1, &dk);
  if (rc == 0) rc = op_attn_launch(c, dq, dk, *a);
  return op_finish(ws, stream, rc, "ssb_op_attention_ex");
}

}  // extern "C"
