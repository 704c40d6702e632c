// Small (HBM-bound) operators of the path: layer norm, embeddings / gathers, masks, samplers,
// pitch glue, RVQ lookup, NSF source.  All operate on guard-banded ragged rows (common.cuh).
// Row addressing convention: grid.y = utterance b, utt[b] = (row_start, len, tight_offset, 0).
#pragma once
#include "common.cuh"

namespace ssb {

// ---- layout / copies -------------------------------------------------------------------------
// tight [total, C] (ld_t) <-> guarded [rows, C] (ld_g); column windows via pointer offset + ld.
int pack_rows(Ctx&, const SeqDev&, const float* tight, int ld_t, float* guarded, int ld_g, int C);
int unpack_rows(Ctx&, const SeqDev&, const float* guarded, int ld_g, float* tight, int ld_t, int C);
int pack_rows_i32(Ctx&, const SeqDev&, const int32_t* tight, int32_t* guarded);
int unpack_rows_i32(Ctx&, const SeqDev&, const int32_t* guarded, int32_t* tight);
int fill_rows(Ctx&, const SeqDev&, float* x, int ld, int C, float value);  // valid rows only
// tight[ti*ld + col] = guarded[r*ld + col]
int unpack_cols_i32(Ctx&, const SeqDev&, const int32_t* guarded, int ld, int col, int32_t* tight);

// ---- normalisation / masks ---------------------------------------------------------------------
// y = LN(x) * gamma + beta over C channels, optionally * rowmask.  x,y [rows, ld].
int layernorm_rows(Ctx&, const SeqDev&, const float* x, int ldx, float* y, int ldy, int C, const float* gamma,
                   const float* beta, float eps, const float* rowmask);
// mask[r] = (sum_c |x[r,c]| > 0) ? 1 : 0
int row_nonzero_mask(Ctx&, const SeqDev&, const float* x, int ld, int C, float* mask);
// mask[r] = (x[r,0] != 0)
int col0_nonzero_mask(Ctx&, const SeqDev&, const float* x, int ld, float* mask);
int token_nonzero_mask(Ctx&, const SeqDev&, const int32_t* tok, float* mask);
// pos[r] = cumsum(mask)[r] * mask[r]  (make_positions, padding_idx 0), per utterance
int positions_from_mask(Ctx&, const SeqDev&, const float* mask, int32_t* pos);
// x[r,c] (+)= alpha_ptr[0] * table[pos[r], c]
int add_positional(Ctx&, const SeqDev&, float* x, int ld, int C, const int32_t* pos, const float* table,
                   int table_rows, const float* alpha_ptr);

// ---- embeddings / gathers ----------------------------------------------------------------------
// x[r,c] = scale * E[tok[r], c]
int embed_rows(Ctx&, const SeqDev&, const int32_t* idx, const float* table, int nrows_table, float scale, float* x,
               int ld, int C, int accumulate);
// note encoder: x = 16*E_note[note] + 16*E_type[type] + (dur * w + b)
int note_encoder(Ctx&, const SeqDev&, const int32_t* note, const int32_t* type, const float* dur, const float* En,
                 const float* Et, const float* w, const float* b, float scale, float* x, int ld, int C, int accumulate);
// out[f, :] = src[ph_row(b) + mel2ph[f] - 1, :] (0 where mel2ph == 0); optional int gather of note -> midi
int expand_states(Ctx&, const SeqDev& frames, const SeqDev& phones, const int32_t* mel2ph, const float* src, int ld_s,
                  float* out, int ld_o, int C, const int32_t* note, int32_t* midi, float* tgt_nonpad);
// out = (sum of up to 4 matrices + up to 3 per-utterance vectors [B, C]) * rowmask
struct CombineArgs {
  const float* m[4] = {nullptr, nullptr, nullptr, nullptr};
  int ldm[4] = {0, 0, 0, 0};
  const float* v[3] = {nullptr, nullptr, nullptr};  // [B, C]
  const float* rowmask = nullptr;
  float* out = nullptr;
  int ldo = 0;
  int C = 0;
};
int combine_rows(Ctx&, const SeqDev&, const CombineArgs&);

// y[r,c] = x[r,c] * mask[r] + rowscalar[r]   (LocalStyleAdaptor: wn_out * mask + ref_f0, lse.py:110,121-123)
int scale_mask_add_rowscalar(Ctx&, const SeqDev&, const float* x, int ldx, int C, const float* mask,
                             const float* rowscalar, float* y, int ldy);
// out[r, 0:C] = z[r, :], out[r, C:2C] = table[pos[r], :]   (cat[style, positions], stylesinger.py:199-200)
int concat2_pos(Ctx&, const SeqDev&, const float* z, int C, const int32_t* pos, const float* table, int table_rows,
                float* out, int ldo);
// g[r, :] = cat[coarse(80) | dec(256) | spk[b](256) | emo[b](256) | style(256)]   (stylesinger.py:314-326), leaving out
// the segments whose pointer is null (dec, emo, style) and packing the rest in that order; ldo = the width that leaves
int concat_cond(Ctx&, const SeqDev&, const float* coarse, const float* dec, const float* spk, const float* emo,
                const float* style, float* out, int ldo);
// x[r, c] = min(max(x, lo), hi) on valid rows
int clip_rows(Ctx&, const SeqDev&, float* x, int ld, int C, float lo, float hi);

// ---- duration ------------------------------------------------------------------------------------
// dur[p] = max(rint(exp(x[p]) - 1), 0) * nonpad
int dur_from_logits(Ctx&, const SeqDev& phones, const float* logdur, const float* nonpad, int32_t* dur);
// mel2ph for frames layout from dur (phones layout): 1-based phone index per frame
int length_regulate(Ctx&, const SeqDev& frames, const SeqDev& phones, const int32_t* dur, int32_t* mel2ph);

// ---- RVQ (a11) -------------------------------------------------------------------------------------
// x [rows, 256] -> quant [rows,256] = x + (agg - x), codes int32 [rows, depth]; codebooks [depth][n_embed][256]
int rvq_lookup(Ctx&, const SeqDev&, const float* x, int ldx, const float* codebooks, const float* cb_norm2,
               int n_embed, int depth, float* quant, int ldq, int32_t* codes);
int codebook_norms(Ctx&, const float* codebooks, int n, float* out);  // ||c||^2 for n rows of 256

// ---- samplers (a14, a19) ------------------------------------------------------------------------------
// x = sqrt_ac * norm_spec(coarse) + sqrt_1m_ac * noise ; coarse == null (ProDiff): x = noise.  Null noise draws Philox
// stream_id with the key and counter base of each utterance's entry of `rng` (the layout's SeqDev::rng); so do the
// other samplers.
int mel_q_sample(Ctx&, const SeqDev&, const float* coarse, int ldc, const float* noise /*tight [total,80] or null*/,
                 const float* spec_min, const float* spec_max, float sa, float s1a, float* x, int ldx, const UttRng* rng,
                 uint64_t stream_id);
// one reverse step: x <- c1*clamp(a*x - b*eps) + c2*x + sigma*noise
struct PlmsArgs {  // one PLMS update over [rows, 80] guarded buffers (see k_plms_update)
  const float* x = nullptr;      // x_t
  float* x_out = nullptr;        // x_{t - interval} (may alias x)
  const float* eps = nullptr;    // current prediction [rows, lde]
  int lde = 0;
  const float *h1 = nullptr, *h2 = nullptr, *h3 = nullptr;  // previous predictions, newest first (null: unused)
  float w0 = 1.f, w1 = 0.f, w2 = 0.f, w3 = 0.f, den = 1.f;
  float a_t = 0.f, a_prev = 0.f;  // alphas_cumprod[t], alphas_cumprod[max(t - interval, 0)]
  float* hist_out = nullptr;     // receives eps (null: the update is the first step's trial x_pred)
};
int plms_update(Ctx&, const SeqDev&, const PlmsArgs&);
int mel_p_sample(Ctx&, const SeqDev&, float* x, int ldx, const float* eps, int lde, const float* noise,
                 const float* tab /*dev ptr to 8 floats for this t*/, const UttRng* rng, uint64_t stream_id,
                 bool clip = true /*false: ProDiff, x0 unclipped*/);
int mel_denorm(Ctx&, const SeqDev&, const float* x, int ldx, const float* spec_min, const float* spec_max,
               const float* rowmask, float* mel_tight, int ld);

struct F0StepArgs {
  float* z = nullptr;            // [rows] gaussian state
  int32_t* uv = nullptr;         // [rows] class state (0 voiced / 1 unvoiced)
  const float* out3 = nullptr;   // [rows, ld3]: (eps, logit0, logit1)
  int ld3 = 4;
  const float* lo = nullptr;     // [rows] dyn clip
  const float* hi = nullptr;
  const float* gnoise = nullptr; // tight [total] or null
  const float* unoise = nullptr; // tight [total, 2] or null
  const float* gtab = nullptr;   // device, 8 floats for this t
  const float* mtab = nullptr;   // device, 8 floats for this t
  int t = 0;
  float log_eps = 0.f;           // fp32 log(1e-30)
  const UttRng* rng = nullptr;                  // Philox keys of the layout (SeqDev::rng)
  uint64_t gauss_stream = 0, unif_stream = 0;  // Philox streams of this step (philox.cuh)
};
int f0_p_sample(Ctx&, const SeqDev&, const F0StepArgs&);
int f0_init(Ctx&, const SeqDev&, float* z, int32_t* uv, const float* gnoise, const UttRng* rng, uint64_t stream_id);
// DDiffNet input: x[r, c<C/2] = f0*w+b ; x[r, c>=C/2] = E_uv[uv]; y = x + d0
int ddiff_input(Ctx&, const SeqDev&, const float* z, const int32_t* uv, const float* w, const float* b, const float* Euv,
                const float* d0, float* x, float* y, int C, __half* yh = nullptr, __half* yl = nullptr);

// ---- pitch glue (a15) -----------------------------------------------------------------------------------
int midi_clip_band(Ctx&, const SeqDev&, const int32_t* midi, float* lo, float* hi);
// pred[r] = ((f0a+f0s)/2 in log2Hz, (uva+uvs)/2) ; f0_denorm ; coarse bin ; all tight outputs optional
struct PitchGlueArgs {
  const float* za = nullptr; const int32_t* uva = nullptr;  // agnostic sampler output (normalised f0, uv class)
  const float* zs = nullptr; const int32_t* uvs = nullptr;  // specific
  const int32_t* midi = nullptr;
  const int32_t* mel2ph = nullptr;
  const float* f0_in = nullptr;   // optional teacher-forced f0 (log2 Hz) guarded [rows]
  const float* uv_in = nullptr;   // optional teacher-forced uv
  float* pitch_pred = nullptr;    // guarded [rows, 2]
  float* f0_denorm = nullptr;     // guarded [rows]
  int32_t* pitch = nullptr;       // guarded [rows] coarse bin
};
int pitch_glue(Ctx&, const SeqDev&, const PitchGlueArgs&);
// f0_gen 'conv': pred[r] = ps/2 + pa/2 of the two PitchPredictor outputs (log2 Hz, uv logit) ; f0_denorm ; coarse bin
struct PitchGlueConvArgs {
  const float* pa = nullptr;      // guarded [rows, 2]: pitch_predictor output (domain agnostic)
  const float* ps = nullptr;      // guarded [rows, 2]: pitch_inpainter_predictor output (domain specific)
  const int32_t* mel2ph = nullptr;
  const float* f0_in = nullptr;   // optional teacher-forced f0 (log2 Hz) guarded [rows]
  const float* uv_in = nullptr;   // optional teacher-forced uv
  float* pitch_pred = nullptr;    // guarded [rows, 2]
  float* f0_denorm = nullptr;     // guarded [rows]
  int32_t* pitch = nullptr;       // guarded [rows] coarse bin
};
int pitch_glue_conv(Ctx&, const SeqDev&, const PitchGlueConvArgs&);

// ---- vocoder helpers (a20, a21) ---------------------------------------------------------------------------
// harmonic source: f0 frames [rows1] -> har [rows256] (guarded at rate 256); Philox keys: s1.rng (initial phase),
// s256.rng (source noise)
int nsf_source(Ctx&, const SeqDev& s1, const SeqDev& s256, const float* f0, const float* lin_w, const float* lin_b,
               const float* rand_ini /*[B,9] or null*/, const float* noise /*tight [total*256, 9] or null*/,
               float* har, double* scratch, int upp, float sr);
size_t nsf_scratch_doubles(const SeqDev& s256);
// x[r, n] += b[n] + sum_j w[n][j] * har[r*s - s/2 + j]   (noise_convs[i], kernel 2s stride s; s==1: kernel 1)
int noise_conv_add(Ctx&, const SeqDev& sx, const SeqDev& s256, float* x, int ld, int C, const float* har, const float* w,
                   const float* b, int s, __half* ph = nullptr, __half* pl = nullptr, float plane_slope = 0.1f,
                   const float* wt = nullptr);  // wt: the weights as [K, C] -> tiled kernel
// wav[tight] = tanh(x[r,0])
int tanh_out(Ctx&, const SeqDev&, const float* x, int ld, float* wav_tight);
// wav = tanh(conv_post(leaky_relu(x, slope))) for a 1-output-channel conv packed as W[taps][C][npad] (column 0)
int conv_post_tanh(Ctx&, const SeqDev&, const float* x, int ld, int C, int taps, int center, const float* W, int npad,
                   const float* bias, float slope, float* wav_tight);
// mask/clip mel (inference/StyleSinger.py:56-58) in place on guarded rows; f0 masked the same way
int mel_postprocess(Ctx&, const SeqDev&, float* mel, int ld, float* f0, float vmin, float vmax);

int mel_postprocess_flat(cudaStream_t st, float* mel, int64_t n, float vmin, float vmax, int32_t* cnt);

}  // namespace ssb
