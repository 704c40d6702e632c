/* stylesinger_b200 — C ABI of the H100-native StyleSinger hot path (libstylesinger_b200.so).
 *
 * The reference (AaronZ345/StyleSinger) is pure Python/PyTorch and has NO FFI of its own
 * (SURVEY.md §8b); its extension points are Python classes and registries.  This header is the
 * boundary a binding for that path attaches to: each entry point replaces one reference interface,
 * cited as file:line of /root/reference.  INTEGRATION.md shows the ctypes stubs and the
 * reference-side registrations (DIFF_DECODERS / FS_ENCODERS / FS_DECODERS / register_vocoder).
 *
 * Conventions
 *  - plain C: pointers + sizes, no torch / C++ types.  `stream` is a cudaStream_t passed as void*.
 *  - all DEVICE tensors are fp32 (or int32) row-major and "tight packed": a batch of B utterances
 *    of lengths L_b is one [sum L_b, C] matrix; `*_offsets` are HOST int32 arrays of B+1 prefix
 *    sums.  Every utterance is processed with true-length (the reference's B=1) semantics —
 *    with injected noise, results do not depend on batch composition.
 *  - the caller owns every device buffer including the workspace (`*_workspace_bytes`); entry
 *    points enqueue on `stream`, never allocate device memory and never synchronise — except
 *    ssb_model_create / ssb_vocoder_create / ssb_model_set_schedule, which own the packed weights.
 *  - return 0 on success, negative on error with a message in ssb_last_error() (thread-local).
 *  - noise: NULL noise pointers select the in-kernel counter-based generator (Philox);
 *    non-NULL pointers inject the noise explicitly (parity mode; SURVEY.md A.10 draw order).
 *    Philox has two modes, which draw the same streams (csrc/philox.cuh) under different keys and counters:
 *     - one seed per call (`seed`, the default): every draw is keyed by `seed` and counted by the tight
 *       row of the whole call (frame, or sample for the vocoder source), and the vocoder's initial
 *       phases by the utterance index; the persistent mel groups (ssb_model_set_persistent_groups) key
 *       group g by seed + 0x9E3779B97F4A7C15 g and count rows inside the group.  An utterance's noise
 *       therefore depends on the batch it is in.
 *     - one seed per utterance (ssb_acoustic_forward_keyed, ssb_hifigan_generate_keyed): utterance b's
 *       draws are keyed by utt_seeds[b] and counted from its own first row, with initial-phase stream
 *       index 0, and nothing is re-seeded per group.  Each draw is bit-for-bit the draw of a B = 1
 *       call with seed = utt_seeds[b], whatever else the batch holds.
 *    The standalone sampler entries (ssb_mel_diffusion_sample[_plms], ssb_mel_prodiff_sample,
 *    ssb_f0_diffusion_sample) have only the per-call mode.
 */
#ifndef STYLESINGER_B200_H
#define STYLESINGER_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ssb_model ssb_model_t;     /* packed StyleSinger acoustic model (immutable after create) */
typedef struct ssb_vocoder ssb_vocoder_t; /* packed HiFi-GAN(-NSF) generator */
typedef struct ssb_melspec ssb_melspec_t; /* STFT + mel filterbank of the reference-audio front-end */
typedef struct ssb_lstm_encoder ssb_lstm_encoder_t; /* LSTM utterance encoder of the reference-audio front-end (emo_embed) */
typedef struct ssb_wav_denoise ssb_wav_denoise_t; /* spectral-subtraction denoiser of the vocoder output (vocoder_denoise_c) */

/* One named fp32 HOST tensor of a reference state_dict (names exactly as in the reference's
 * checkpoints: utils/commons/ckpt_utils.py:26-67 loads state_dict['model']). */
typedef struct {
  const char* name;
  const float* data;
  int32_t ndim;
  int64_t shape[4];
} ssb_tensor_desc;

/* egs/stylesinger.yaml keys the kernels are specialised on (reference egs/stylesinger.yaml:10-141). */
typedef struct {
  int32_t hidden_size;     /* 256 */
  int32_t enc_layers, dec_layers;           /* 4, 4 */
  int32_t enc_ffn_kernel, dec_ffn_kernel;   /* 9, 9 */
  int32_t dur_layers, dur_kernel;           /* 2, 3 */
  int32_t n_tokens;                         /* len(phone dictionary) */
  int32_t n_rq, rq_depth;                   /* 128, 4 */
  int32_t mel_channels, mel_layers, mel_cycle; /* residual_channels 256, residual_layers 20, dilation_cycle_length 4 */
  int32_t f0_channels, f0_layers, f0_cycle;    /* 192, 10, 4 */
  int32_t mel_bins;                         /* 80 */
} ssb_hparams;

/* HiFi-GAN generator config (checkpoints/hifigan/config.yaml keys read at
 * tasks/tts/vocoder_infer/hifigan_nsf.py:48-60, modules/hifigan/hifigan_nsf.py:104-142). */
typedef struct {
  int32_t n_up;
  int32_t up_rates[8];
  int32_t up_kernels[8];
  int32_t initial_channel;
  int32_t n_res;
  int32_t res_kernels[4];
  int32_t res_dilations[4][3];
  int32_t use_pitch_embed; /* NSF harmonic source */
  int32_t sample_rate;
} ssb_vocoder_config;

/* ssb_vocoder_config plus the ResBlock type (config key 'resblock', modules/hifigan/hifigan_nsf.py:115):
 *   1: ResBlock1 (:30-66), 3 dilations per block (res_dilations[j][0..2]), convs1.{m} / convs2.{m} per dilation;
 *   2: ResBlock2 (:69-90), 2 dilations per block (res_dilations[j][0..1]; [j][2] is unread), convs.{m} per dilation.
 * This covers the three published HiFi-GAN layouts: V1 (512 initial channels, ResBlock1), V2 (128, ResBlock1) and
 * V3 (256, ResBlock2). */
typedef struct {
  int32_t n_up;
  int32_t up_rates[8];
  int32_t up_kernels[8];
  int32_t initial_channel;
  int32_t n_res;
  int32_t res_kernels[4];
  int32_t res_dilations[4][3];
  int32_t use_pitch_embed;
  int32_t sample_rate;
  int32_t resblock; /* 1 or 2 */
} ssb_vocoder_config_ex;

int ssb_version(void);
const char* ssb_last_error(void);

/* Replaces StyleSinger.__init__ + load_ckpt (modules/StyleSinger/stylesinger.py:46-117,
 * utils/commons/ckpt_utils.py:26-67).  Extra host-computed constant expected in `tensors`:
 *   "__pos_table" [rows,256]: SinusoidalPositionalEmbedding.get_embedding(rows,256,0)
 *   (modules/commons/common_layers.py:111-127), rows >= max sequence length + 2. */
int ssb_model_create(ssb_model_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_hparams* hp);
void ssb_model_free(ssb_model_t* m);

/* hparams['decoder'] (modules/StyleSinger/stylesinger.py:98-117,176-184): which mel decoder the model was built with. */
#define SSB_MEL_DECODER_DIFFSINGER 0 /* FFT decoder -> mel_out -> ln_proj -> DDPM over postdiff.denoise_fn (the default) */
#define SSB_MEL_DECODER_PRODIFF 1    /* ProDiff teacher (modules/diff/prodiff.py:59-232): decoder_inp is the condition of an
                                      * x0-predicting sampler over diff_decoder.denoise_fn; no FFT decoder / mel_out / ln_proj */
#define SSB_MEL_DECODER_FFT 2        /* FastSpeech 2 decoder alone (stylesinger.py:185-186, fs2.py:233-237): mel_out(decoder(
                                      * decoder_inp)) * tgt_nonpadding is the mel; no ln_proj, no mel DiffNet, no diffusion */
/* ssb_model_create with the mel decoder chosen: ssb_model_create(...) == ssb_model_create_ex(..., SSB_MEL_DECODER_DIFFSINGER).
 * PRODIFF loads the mel DiffNet from "diff_decoder.denoise_fn.*" and needs no "postdiff.*" / "ln_proj.*" ("decoder.*" is
 * still packed for ssb_fft_decoder; "mel_out.*" and the "diff_decoder.*" buffers are accepted and ignored).  The schedule
 * (ssb_model_set_schedule, which = 0) is then the ProDiff table: slots {0, -1, post_coef1, post_coef2, sigma, -, -,
 * alphas_cumprod} of the vpsde schedule (prodiff.py:11-13,69-117).  An unknown mel_decoder fails before any CUDA call. */
int ssb_model_create_ex(ssb_model_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_hparams* hp,
                        int32_t mel_decoder);

/* hparams['f0_gen'] (modules/StyleSinger/stylesinger.py:66-82,223-228): which F0 generator the model was built with. */
#define SSB_F0_GEN_GMDIFF 0 /* two 100-step Gaussian-multinomial diffusion samplers over gm_diffnet(_inpainte) (the default) */
#define SSB_F0_GEN_CONV 1   /* two FastSpeech-2 PitchPredictors (modules/fastspeech/tts_modules.py:191-234): deterministic */
/* ssb_model_create_ex with the F0 generator chosen as well: ssb_model_create_ex(..., d) ==
 * ssb_model_create_ex2(..., d, SSB_F0_GEN_GMDIFF).  CONV loads "pitch_predictor.*" (domain agnostic) and
 * "pitch_inpainter_predictor.*" (domain specific): per predictor conv.{0..4}.1.weight [256,256,k] (k odd, (k-1)/2 <= 16) /
 * .bias, conv.{i}.3.weight / .bias (LayerNorm), linear.weight [2,256] / .bias and pos_embed_alpha [1]; "gm_diffnet*" and
 * "f0_gen*" are neither required nor packed.  On a CONV model the F0 schedule (ssb_model_set_schedule, which = 1),
 * ssb_f0_diffusion_sample, ssb_denoiser_eval(which = 1 / 2) and F0 noise pointers in ssb_acoustic_inputs are errors; on a
 * GMDIFF model ssb_pitch_predictor is.  An unknown mel_decoder or f0_gen fails before any CUDA call. */
int ssb_model_create_ex2(ssb_model_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_hparams* hp,
                         int32_t mel_decoder, int32_t f0_gen);

/* The boolean model switches of egs/stylesinger.yaml's "choices of models" block and hparams['use_txt_cond'], each 0 or 1
 * (modules/StyleSinger/stylesinger.py:53-64,92-110,119-187,313-331):
 *   emo          emo_embed_proj (:53-54); emo is added to dur_inp (:136-137), pitch_inp_domain_specific (:159-160),
 *                decoder_inp (:168-169) and concatenated into the ln_proj input (:321-323).
 *   style        style_extractor / l1 / align (:61-64); get_style runs (:149-151) and style is added to
 *                pitch_inp_domain_specific (:161-162), decoder_inp (:170-171) and concatenated into ln_proj's input (:324-326).
 *   umln         norm (DistributionUncertainty, :57-58): the identity at inference (umln.py:49-50), so the switch only
 *                decides whether "norm.affine_layer.*" belongs to the checkpoint.  It is never packed.
 *   use_txt_cond decoder_inp concatenated into ln_proj's input (:94-95,317-318).
 * ln_proj's input (DiffSinger models) is cat[coarse_mel, decoder_inp if use_txt_cond, spk, emo if emo, style if style],
 * 80 + 256 (1 + use_txt_cond + emo + style) columns. */
typedef struct {
  int32_t emo, style, umln, use_txt_cond;
} ssb_model_switches;

/* ssb_model_create_ex2 with the model switches chosen: ssb_model_create_ex2(..., d, f) == ssb_model_create_ex3(..., d, f,
 * {1, 1, 1, 1}).  Only the modules the switches build are read and packed; keys of switched-off modules are ignored, as
 * the reference's load_ckpt(..., strict=False) ignores them (inference/StyleSinger.py:38).  On a model without emo,
 * in->emo_embed may be NULL and is never read; without style, in->ref_offsets / ref_mels / ref_f0 may be NULL and are never
 * read, no style adaptor, RVQ or aligner runs and its buffers are not taken from the workspace.  Asking such a model for
 * out->emo_proj (no emo), out->style or out->rq_codes (no style) is an error, and so are ssb_get_style and ssb_rvq_lookup
 * (no style).  Fails, naming the cause and leaving *out NULL, before anything is allocated when a switch is not 0 / 1, or
 * (DiffSinger models) when "ln_proj.weight" is not [256, 80 + 256 (1 + use_txt_cond + emo + style)]. */
int ssb_model_create_ex3(ssb_model_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_hparams* hp,
                         int32_t mel_decoder, int32_t f0_gen, const ssb_model_switches* switches);

/* ssb_model_create_ex3 with the speaker input chosen: ssb_model_create_ex3(..., d, f, sw) == ssb_model_create_ex4(..., d, f,
 * sw, 0).  hparams['use_spk_id'] (modules/fastspeech/fs2.py:37-43): with use_spk_id = 1, "spk_embed_proj.weight" [rows, 256]
 * (Embedding(num_spk + 1, 256), no bias) is packed as a lookup table, and every acoustic entry (ssb_acoustic_forward,
 * ssb_acoustic_forward_keyed, ssb_predict_durations and their *_workspace_bytes) reads in->spk_ids instead of
 * in->spk_embed: spk = table[spk_ids[b]] (stylesinger.py:130), out->spk_proj returns those rows.  The ids are checked on the
 * host against [0, rows) before anything is launched; NULL spk_ids is an error.  Everything downstream of spk is unchanged.
 * With use_spk_id = 0 "spk_embed_proj.weight" is the Linear(256, 256) over in->spk_embed (and .bias is required).
 * "spk_embed_f0.*" / "spk_embed_dur.*" (use_split_spk_id) are never read.  use_spk_id combines with every mel decoder, F0
 * generator and switch.
 * SSB_MEL_DECODER_FFT models pack "decoder.*" and "mel_out.*"; "postdiff.*", "ln_proj.*" and "diff_decoder.*" are neither
 * required nor read.  Their forward is the FFT decoder and mel_out with the tgt_nonpadding row mask into out->mel_out
 * (out->coarse_mel, when asked for, holds the same values); skip_mel_diffusion has no effect, pndm_speedup is ignored as
 * the reference ignores it.  On an FFT model these are errors, refused with a message before any launch: out->diff_cond,
 * a non-NULL in->mel_noise, ssb_model_set_schedule(which = 0), ssb_model_set_mel_k_step (any K),
 * ssb_mel_diffusion_sample[_plms], ssb_mel_prodiff_sample and ssb_denoiser_eval(which = 0).  ssb_model_set_mel_precision
 * is accepted and changes nothing (there is no mel DiffNet).  Fails, naming the cause and leaving *out NULL, before anything
 * is allocated when use_spk_id is not 0 / 1 or mel_decoder / f0_gen is unknown. */
int ssb_model_create_ex4(ssb_model_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_hparams* hp,
                         int32_t mel_decoder, int32_t f0_gen, const ssb_model_switches* switches, int32_t use_spk_id);

/* Diffusion schedules (GaussianDiffusion.__init__ modules/diff/shallow_diffusion_tts.py:68-122;
 * GaussianMultinomialDiffusion.__init__ modules/diff/gaussian_multinomial_diffusion.py:208-284).
 * which: 0 = mel denoiser, 1 = both F0 denoisers.  Host arrays:
 *   step_emb [T, C]   SinusoidalPosEmb(t) (modules/diff/net.py:31-44), C = residual channels
 *   gauss_tab [T, 8]  {sqrt_recip_ac, sqrt_recipm1_ac, post_coef1, post_coef2, sigma, sqrt_ac, sqrt_1m_ac, 0}
 *   multi_tab [T, 8]  {log_alpha_t, log_1m_alpha_t, log_cumprod_alpha_{t-1}, log_1m_cumprod_alpha_{t-1}, ...} (which==1)
 * Builds the per-layer step-bias table [T, L, C] on the device.  Synchronises `stream`. */
int ssb_model_set_schedule(ssb_model_t* m, int32_t which, int32_t T, const float* step_emb, const float* gauss_tab,
                           const float* multi_tab, void* stream);

/* hparams['K_step'] of the DiffSinger mel sampler (shallow diffusion; GaussianDiffusion.__init__ and
 * DiffusionDecoder.forward, modules/diff/shallow_diffusion_tts.py:92,297-304): x_K = q_sample(norm_spec(coarse), K-1) on
 * the T-step schedule, then K reverse steps t = K-1 .. 0 (the PLMS sampler: t0 = the largest multiple of the interval
 * below K).  K = 0 (the default) follows the schedule's T.  Every mel-sampler entry (ssb_acoustic_forward,
 * ssb_mel_diffusion_sample, ssb_mel_diffusion_sample_plms and their *_workspace_bytes) then uses K_eff = K ? K : T and
 * fails if K_eff > T.  K < 0, and any K on a PRODIFF model (ProDiffusion.forward never reads K_step), are errors.
 * Philox mode: step t draws the same stream at every K. */
int ssb_model_set_mel_k_step(ssb_model_t* m, int32_t K);

/* Inputs of StyleSinger.forward(..., infer=True) (modules/StyleSinger/stylesinger.py:119-187). */
typedef struct {
  int32_t B;
  const int32_t* ph_offsets;    /* host [B+1] */
  const int32_t* frame_offsets; /* host [B+1]; required by ssb_acoustic_forward */
  const int32_t* ref_offsets;   /* host [B+1]; NULL allowed on a model without style (ssb_model_create_ex3) */
  const int32_t* txt_tokens;    /* dev [sumP] */
  const int32_t* note;          /* dev [sumP] */
  const int32_t* note_type;     /* dev [sumP] */
  const float* note_dur;        /* dev [sumP] */
  const float* spk_embed;       /* dev [B,256] */
  const float* emo_embed;       /* dev [B,256]; NULL allowed on a model without emo */
  const float* ref_mels;        /* dev [sumR,80]; NULL allowed on a model without style */
  const float* ref_f0;          /* dev [sumR]; NULL allowed on a model without style */
  const int32_t* mel2ph;        /* dev [sumF] 1-based phone index per frame, or NULL -> use `dur` */
  const int32_t* dur;           /* dev [sumP] frames per phone (from ssb_predict_durations), or NULL */
  const float* f0;              /* dev [sumF] optional teacher-forced log2-Hz f0 (forward kwarg f0) */
  const float* uv;              /* dev [sumF] optional teacher-forced uv */
  const float* f0_gauss_noise[2]; /* dev [(T_f0+1), sumF]: z init then one per step t=T-1..0; NULL -> Philox */
  const float* f0_unif_noise[2];  /* dev [T_f0, sumF, 2] */
  const float* mel_noise;         /* dev [(K+1), sumF, 80]: the q_sample draw, then one per step t = K-1 .. 0
                                   * (K = ssb_model_set_mel_k_step's K_eff; T on a PRODIFF model) */
  uint64_t seed;
  int32_t skip_mel_diffusion;     /* 1: stop after the coarse mel / diff_cond */
  int32_t pndm_speedup;           /* 0: DDPM ancestral sampling, K steps (the StyleSinger default, DiffusionDecoder.forward);
                                   * k in [1, K): PLMS with iteration interval k (hparams['pndm_speedup'],
                                   * modules/diff/shallow_diffusion_tts.py:164-197,254-260): K / k (+1) denoiser evaluations */
  const int32_t* spk_ids;         /* host [B]: speaker ids, read only on a model created with use_spk_id = 1
                                   * (ssb_model_create_ex4), which then never reads spk_embed; other models never read it */
} ssb_acoustic_inputs;

/* Outputs (all optional except mel_out/f0_denorm when diffusion runs); device, tight packed. */
typedef struct {
  float* mel_out;       /* [sumF,80]   ret['mel_out'] */
  float* f0_denorm;     /* [sumF]      ret['f0_denorm'] (Hz) */
  float* encoder_out;   /* [sumP,256]  encoder(txt)+note_encoder */
  float* style;         /* [sumF,256]  ret['style'] */
  int32_t* rq_codes;    /* [sumR,4]    RVQ indices */
  float* pitch_pred;    /* [sumF,2]    ret['pitch_pred'] */
  float* decoder_inp;   /* [sumF,256]  ret['decoder_inp'] */
  float* coarse_mel;    /* [sumF,80]   FFT-decoder mel before diffusion */
  float* diff_cond;     /* [sumF,256]  ln_proj(cat[...]) */
  int32_t* mel2ph;      /* [sumF] */
  float* spk_proj;      /* [B,256] ret['spk_embed'] */
  float* emo_proj;      /* [B,256] ret['emo_embed'] */
} ssb_acoustic_outputs;

/* FastSpeech2.add_dur -> DurationPredictor.inference (modules/fastspeech/fs2.py:151-174,
 * modules/fastspeech/tts_modules.py:105-130): dur[p] = clamp(round(exp(x)-1), 0).
 * The host reads `dur_out` back to size the frame axis (the reference syncs here too). */
size_t ssb_durations_workspace_bytes(const ssb_model_t* m, const ssb_acoustic_inputs* in);
int ssb_predict_durations(const ssb_model_t* m, const ssb_acoustic_inputs* in, int32_t* dur_out, float* logdur_out,
                          void* workspace, size_t workspace_bytes, void* stream);

/* StyleSinger.forward(infer=True, global_steps > diff_start): rows a1-a19 of SURVEY.md §8.
 * On a PRODIFF model (stylesinger.py:174-177): decoder_inp goes straight to the ProDiff sampler (no FFT decoder, mel_out or
 * ln_proj); pndm_speedup is ignored like the reference ignores it; asking for coarse_mel or diff_cond is an error.
 * On a CONV F0 model (inpaint_pitch, stylesinger.py:216-247): pitch_pred = specific/2 + agnostic/2 of the two
 * PitchPredictors (always run, also with teacher-forced f0); f0 = pitch_pred[..., 0] in log2 Hz with no MIDI band or
 * de-normalisation, uv = pitch_pred[..., 1] > 0, rests not forced unvoiced; no F0 noise is drawn (mel_noise is then the
 * forward's only noise), and non-NULL f0_gauss_noise / f0_unif_noise are an error. */
size_t ssb_acoustic_workspace_bytes(const ssb_model_t* m, const ssb_acoustic_inputs* in);
int ssb_acoustic_forward(const ssb_model_t* m, const ssb_acoustic_inputs* in, const ssb_acoustic_outputs* out,
                         void* workspace, size_t workspace_bytes, void* stream);
/* ssb_acoustic_forward with one Philox seed per utterance: utt_seeds (HOST [B], required) keys utterance b's draws, so
 * its outputs are those of a B = 1 ssb_acoustic_forward with seed = utt_seeds[b] (up to the GEMM path a batch of that size
 * takes).  in->seed is ignored; injected noise (mel_noise, f0_gauss_noise, f0_unif_noise) is an error.  The workspace is
 * ssb_acoustic_workspace_bytes(m, in). */
int ssb_acoustic_forward_keyed(const ssb_model_t* m, const ssb_acoustic_inputs* in, const uint64_t* utt_seeds,
                               const ssb_acoustic_outputs* out, void* workspace, size_t workspace_bytes, void* stream);

/* DiffusionDecoder.forward(infer=True) alone (modules/diff/shallow_diffusion_tts.py:284-307):
 * cond [sumF,256], coarse [sumF,80] -> mel [sumF,80].  DiffSinger models only (the PLMS entry point too).
 * noise [(K+1),sumF,80] = the q_sample draw, then one per step t = K-1 .. 0 (K: ssb_model_set_mel_k_step), or NULL (Philox). */
size_t ssb_mel_diffusion_workspace_bytes(const ssb_model_t* m, const int32_t* frame_offsets, int32_t B);
int ssb_mel_diffusion_sample(const ssb_model_t* m, const float* cond, const float* coarse_mel,
                             const int32_t* frame_offsets, int32_t B, const float* noise, uint64_t seed,
                             float* mel_out, void* workspace, size_t workspace_bytes, void* stream);

/* PLMS / PNDM sampler over the same DiffNet (SURVEY.md section 8f, f2): GaussianDiffusion.p_sample_plms driven by the
 * `pndm_speedup` loop of GaussianDiffusion.forward (modules/diff/shallow_diffusion_tts.py:164-197,254-260).
 * interval = hparams['pndm_speedup'], in [1, K) (K: ssb_model_set_mel_k_step); q_noise [sumF,80] (tight) is the single
 * q_sample draw (at K-1), NULL = in-kernel Philox. */
size_t ssb_mel_diffusion_plms_workspace_bytes(const ssb_model_t* m, const int32_t* frame_offsets, int32_t B);
int ssb_mel_diffusion_sample_plms(const ssb_model_t* m, const float* cond, const float* coarse_mel,
                                  const int32_t* frame_offsets, int32_t B, const float* q_noise, uint64_t seed,
                                  int32_t interval, float* mel_out, void* workspace, size_t workspace_bytes, void* stream);

/* ProDiffusion.forward(cond, infer=True) alone (modules/diff/prodiff.py:204-222, p_sample :143-148, q_posterior_sample
 * :135-141), PRODIFF models only: x_T = randn; per step x0 = denoise_fn(x_t, t, cond) (no eps -> x0 conversion, no clip),
 * x_{t-1} = posterior mean + [t > 0] exp(0.5 logvar) noise; mel = x_0 (denorm_spec is the identity, no mask).
 * cond [sumF,256] (decoder_inp); noise [(T+1),sumF,80] = the x_T draw then one per step t = T-1..0, or NULL (Philox). */
size_t ssb_mel_prodiff_workspace_bytes(const ssb_model_t* m, const int32_t* frame_offsets, int32_t B);
int ssb_mel_prodiff_sample(const ssb_model_t* m, const float* cond, const int32_t* frame_offsets, int32_t B,
                           const float* noise, uint64_t seed, float* mel_out, void* workspace, size_t workspace_bytes,
                           void* stream);

/* One denoiser evaluation, DiffNet.forward / DDiffNet.forward (modules/diff/net.py:107-130,242-266).
 * which: 0 mel (x [sumF,80] -> eps [sumF,80]); 1 / 2 F0 agnostic / specific (x = f0 [sumF], uv int32 [sumF]
 * -> out [sumF,3]). */
int ssb_denoiser_eval(const ssb_model_t* m, int32_t which, const float* x, const int32_t* uv, int32_t t,
                      const float* cond, const int32_t* frame_offsets, int32_t B, float* out, void* workspace,
                      size_t workspace_bytes, void* stream);

/* GaussianMultinomialDiffusion.sample (modules/diff/gaussian_multinomial_diffusion.py:921-942).
 * which: 0 agnostic net (gm_diffnet), 1 specific (gm_diffnet_inpainte). cond [sumF,256], clip lo/hi [sumF]
 * -> f0_norm [sumF] (normalised), uv int32 [sumF]. */
int ssb_f0_diffusion_sample(const ssb_model_t* m, int32_t which, const float* cond, const float* clip_lo,
                            const float* clip_hi, const int32_t* frame_offsets, int32_t B, const float* gauss_noise,
                            const float* unif_noise, uint64_t seed, float* f0_norm_out, int32_t* uv_out,
                            void* workspace, size_t workspace_bytes, void* stream);

/* PitchPredictor.forward(xs) alone (modules/fastspeech/tts_modules.py:191-234), CONV F0 models only.  which: 0
 * pitch_predictor (run on decoder_inp * tgt_nonpadding), 1 pitch_inpainter_predictor (run on (decoder_inp + spk + emo +
 * style) * tgt_nonpadding), stylesinger.py:155-163,223-225.  x [sumF,256] -> out [sumF,2] (log2-Hz f0, uv logit).  Per
 * utterance: x += pos_embed_alpha * sinusoid[make_positions(x[:, 0])] (a row whose channel 0 is exactly 0 gets position 0
 * and does not advance the count), then 5 x (zero SAME pad, Conv1d 256 -> 256 + bias, ReLU, LayerNorm over channels eps
 * 1e-5), then Linear 256 -> 2; no mask anywhere (the reference applies none). */
size_t ssb_pitch_predictor_workspace_bytes(const ssb_model_t* m, const int32_t* frame_offsets, int32_t B);
int ssb_pitch_predictor(const ssb_model_t* m, int32_t which, const float* x, const int32_t* frame_offsets, int32_t B,
                        float* out, void* workspace, size_t workspace_bytes, void* stream);

/* Per-registry drop-ins (SURVEY.md section 8b).  The reference dispatches through FS_ENCODERS / FS_DECODERS
 * (modules/fastspeech/fs2.py:9-18,30-31) and calls StyleSinger.get_style (modules/StyleSinger/stylesinger.py:189-214):
 *  ssb_fft_encoder  = FastspeechEncoder.forward(txt_tokens) (tts_modules.py:326-346): tokens int32 [sumP] -> [sumP,256]
 *                     (embedding * sqrt(H) + sinusoidal positions, FFT blocks, final LayerNorm, padding rows zero);
 *  ssb_fft_decoder  = FastspeechDecoder.forward(x) (tts_modules.py:349-355, FFTBlocks.forward :281-306): x [sumF,256]
 *                     -> [sumF,256], padding mask = rows of x that are all zero;
 *  ssb_get_style    = get_style(decoder_inp, ref_mels, ...) with ret['ref_f0'] (LocalStyleAdaptor + RVQ + l1 +
 *                     ProsodyAligner, lse.py:103-129,59-81): -> style [sumF,256], codes int32 [sumR,depth] (optional).
 * which (workspace query): 0 encoder (offsets = ph_offsets), 1 decoder (offsets = frame_offsets). */
size_t ssb_fft_workspace_bytes(const ssb_model_t* m, int32_t which, const int32_t* offsets, int32_t B);
int ssb_fft_encoder(const ssb_model_t* m, const int32_t* txt_tokens, const int32_t* ph_offsets, int32_t B, float* out,
                    void* workspace, size_t workspace_bytes, void* stream);
int ssb_fft_decoder(const ssb_model_t* m, const float* x, const int32_t* frame_offsets, int32_t B, float* out,
                    void* workspace, size_t workspace_bytes, void* stream);
size_t ssb_get_style_workspace_bytes(const ssb_model_t* m, const int32_t* frame_offsets, const int32_t* ref_offsets, int32_t B);
int ssb_get_style(const ssb_model_t* m, const float* decoder_inp, const int32_t* frame_offsets, const float* ref_mels,
                  const float* ref_f0, const int32_t* ref_offsets, int32_t B, float* style_out, int32_t* codes_out,
                  void* workspace, size_t workspace_bytes, void* stream);

/* RQBottleneck.forward / VQEmbedding.find_nearest_embedding (modules/StyleSinger/RQ.py:262-270,29-55). */
int ssb_rvq_lookup(const ssb_model_t* m, const float* x /*[sumR,256]*/, const int32_t* ref_offsets, int32_t B,
                   float* quant_out /*[sumR,256]*/, int32_t* codes_out /*[sumR,depth]*/, void* workspace,
                   size_t workspace_bytes, void* stream);

/* HifiGanGenerator (modules/hifigan/hifigan_nsf.py:104-178) with weight norm folded at pack time. */
int ssb_vocoder_create(ssb_vocoder_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_vocoder_config* cfg);
void ssb_vocoder_free(ssb_vocoder_t* v);

/* HifiGanGenerator of any ResBlock type (HifiGanGenerator.__init__, modules/hifigan/hifigan_nsf.py:104-142, picks
 * ResBlock1 or ResBlock2 at :115 from the checkpoint's config, tasks/tts/vocoder_infer/hifigan_nsf.py:24-60).
 * ssb_vocoder_create(out, t, n, cfg) == ssb_vocoder_create_ex with the same fields and resblock = 1.
 * ResBlock2 reads "resblocks.{i*n_res+j}.convs.{m}.{weight_g,weight_v,bias}", m = 0, 1 (:72-79), and runs
 * x = convs[m](leaky_relu(x, 0.1)) + x (:82-87).  Stage i has initial_channel / 2^(i+1) channels: a multiple of 32, or
 * 16 or 8 (HiFi-GAN V2's last two stages).  The ResBlock convs of a 16- or 8-channel stage run as 64-channel convs over
 * groups of 64 / C consecutive samples, so the stage's cumulative upsampling rate prod(up_rates[0..i]) must be a multiple
 * of 64 / C.  Fails, naming the cause and leaving *out NULL, before anything is allocated when resblock is not 1 or 2, a
 * read dilation is below 1, or a stage's channel count or rate breaks the rules above. */
int ssb_vocoder_create_ex(ssb_vocoder_t** out, const ssb_tensor_desc* tensors, int32_t n, const ssb_vocoder_config_ex* cfg);

/* HifiGAN.spec2wav / HifiGanGenerator.forward (tasks/tts/vocoder_infer/hifigan_nsf.py:62-75,
 * modules/hifigan/hifigan_nsf.py:144-169).  mel [sumF,80] (already masked/clipped as
 * inference/StyleSinger.py:56-58 does), f0 [sumF] Hz or NULL.  rand_ini [B,9] / src_noise [sumF*hop, 9]:
 * SineGen's torch.rand / torch.randn draws (modules/parallel_wavegan/models/source.py:357,436) or NULL.
 * wav_out [sumF*hop]. */
size_t ssb_vocoder_workspace_bytes(const ssb_vocoder_t* v, const int32_t* frame_offsets, int32_t B);
int ssb_hifigan_generate(const ssb_vocoder_t* v, const float* mel, const float* f0, const int32_t* frame_offsets,
                         int32_t B, const float* rand_ini, const float* src_noise, uint64_t seed, float* wav_out,
                         void* workspace, size_t workspace_bytes, void* stream);
/* ssb_hifigan_generate with one Philox seed per utterance (utt_seeds: HOST [B], required) and no injected noise: utterance
 * b's SineGen draws are those of a B = 1 call with seed = utt_seeds[b].  The workspace is ssb_vocoder_workspace_bytes. */
int ssb_hifigan_generate_keyed(const ssb_vocoder_t* v, const float* mel, const float* f0, const int32_t* frame_offsets,
                               int32_t B, const uint64_t* utt_seeds, float* wav_out, void* workspace,
                               size_t workspace_bytes, void* stream);

/* Select the GEMM path of the denoiser layers: 1 = wgmma tensor cores on fp16 hi/lo split operands
 * (3 MMAs per product, fp32 accumulate; default when available), 0 = fp32 FFMA.  Returns the mode in effect. */
int ssb_model_set_tensor_cores(ssb_model_t* m, int32_t enable);

/* Same switch for the vocoder's ResBlock convs (wide stages with C % 64 == 0, and the grouped 32-, 16- and 8-channel
 * stages). */
int ssb_vocoder_set_tensor_cores(ssb_vocoder_t* v, int32_t enable);

/* Precision of the tensor-core GEMMs (ssb_model_set_mel_precision, ssb_vocoder_set_precision).  SSB_TC_SPLIT (the
 * default): every fp32 operand is carried as fp16 hi/lo planes and each K step issues 3 MMAs (hi*hi + hi*lo + lo*hi, ~22
 * mantissa bits).  SSB_TC_FP16: one MMA on the hi planes alone (operands rounded once to fp16, fp32 accumulation): a third
 * of the MMAs and half the operand bytes, at a stated accuracy cost (README "Single-pass fp16 mode").  It is a choice of
 * speed against accuracy, like K_step, not another path to the same result. */
#define SSB_TC_SPLIT 0
#define SSB_TC_FP16 1
/* The mel DiffNet on every mel sampler that runs it on tensor cores: DDPM (persistent and per-launch, with the hoisted
 * conditioner projection), K_step, PLMS, ProDiff, and ssb_denoiser_eval(which = 0).  Not the F0 samplers, attention, the
 * FFT blocks, the style adaptor / RVQ, the pitch predictors, the front-end or the output denoiser; GEMMs that take the
 * FFMA path (short batches, ssb_model_set_tensor_cores(0)) are unchanged.  An unknown mode fails and changes nothing.
 * Returns 0 on success. */
int ssb_model_set_mel_precision(ssb_model_t* m, int32_t mode);
/* The vocoder's tensor-core GEMMs (every HiFi-GAN layout, with and without NSF): the ups convs and the ResBlock convs
 * that run on tensor cores.  The FFMA convs (conv_pre, conv_post, narrow FFMA stages) are unchanged. */
int ssb_vocoder_set_precision(ssb_vocoder_t* v, int32_t mode);

/* 1 (default): small batches run the whole T-step mel sampler in ONE persistent cooperative kernel launch
 * (csrc/sampler_tc.cu); 0: one launch per GEMM (BASELINE.json configs[4] compares the two). */
int ssb_model_set_persistent(ssb_model_t* m, int32_t enable);
/* 0 (default): batches of more than 48 row tiles (~6 k frames) take the one-launch-per-GEMM path.  1: such batches are
 * split into groups of consecutive utterances of <= 48 row tiles and every group runs the T-step mel sampler
 * (shallow_diffusion_tts.py:303-304) as ONE persistent launch (production RNG mode only; each group draws from its own
 * Philox stream).  This is the "persistent-kernel" arm of BASELINE.json configs[4] at batch 64. */
int ssb_model_set_persistent_groups(ssb_model_t* m, int32_t enable);
/* Decoder FFT blocks (modules/commons/transformer.py TransformerFFNLayer, conv k=9 -> gelu -> linear): run the FFN GEMMs
 * on the tensor-core kernel for batches of >= 1024 frames (default on; 0 keeps them on the fp32 FFMA kernel). Returns the
 * new setting. */
int ssb_model_set_fft_tensor_cores(ssb_model_t* m, int32_t enable);

/* StyleSingerInfer.forward_model glue between model and vocoder (inference/StyleSinger.py:56-58):
 * clips mel [n_frames,80] in place to [vmin, vmax] and counts the frames with sum|mel| > 0 into
 * *nonzero_frames (device int32; the reference drops all-zero frames, which only padding can produce). */
int ssb_mel_postprocess(float* mel, int64_t n_frames, float vmin, float vmax, int32_t* nonzero_frames, void* stream);

/* ---- f3: mel-spectrogram of the reference audio (SURVEY.md section 8f) -------------------------------------------------
 * Replaces utils/audios/__init__.py:36-84 librosa_wav2spec as called by inference/StyleSinger.py:79-92 (process_audio):
 * librosa.stft(center=True, pad_mode="constant", periodic Hann window) -> |.| -> librosa.filters.mel (Slaney scale and
 * normalisation, built inside create) -> log10(max(eps, .)).  fmin / fmax < 0 mean 0 / sample_rate / 2 like the reference.
 * Constraints of the implicit-GEMM formulation: fft_size even, fft_size <= 32 hop_size (16 with reflect centring), hop_size a multiple of 16, n_mels of 4
 * (egs/stylesinger.yaml: 48 kHz, fft 1024, hop 256, win 1024, 80 mels, 20..24000 Hz).  An utterance of n samples yields
 * ssb_melspec_num_frames = 1 + n / hop_size frames.  wav: device fp32, utterances concatenated, sample_offsets: host [B+1];
 * mel_out: device fp32 [sum frames, n_mels].  loud_norm / trim_long_sil of the reference are not implemented (both false in
 * the reference's configuration); the speaker / emotion encoders and the Praat pitch tracker are outside this library. */
int ssb_melspec_create(ssb_melspec_t** out, int32_t sample_rate, int32_t fft_size, int32_t hop_size, int32_t win_length,
                       int32_t n_mels, float fmin, float fmax, float eps);
/* Same front-end with the defaults of librosa.feature.melspectrogram selectable, which is what the emotion encoder's features
 * are (data_gen/tts/emotion/audio.py:43-55: sr 16000, n_fft 400, hop 160, 40 mels, fmin 0, fmax sr / 2): pad_reflect != 0 =
 * np.pad "reflect" centring instead of zeros (reflected as often as the pad needs, like numpy; an empty utterance is refused,
 * as numpy refuses it), power != 0 = |X|^2
 * instead of |X|, take_log == 0 = no log10 / eps.  n_fft need not be a multiple of hop_size here (the frame is embedded in
 * the next multiple of 2 hop_size rows with zero weights).  ssb_melspec_create = (..., 0, 0, 1). */
int ssb_melspec_create_ex(ssb_melspec_t** out, int32_t sample_rate, int32_t fft_size, int32_t hop_size, int32_t win_length,
                          int32_t n_mels, float fmin, float fmax, float eps, int32_t pad_reflect, int32_t power, int32_t take_log);
void ssb_melspec_free(ssb_melspec_t* m);
int32_t ssb_melspec_num_frames(const ssb_melspec_t* m, int64_t n_samples);
size_t ssb_melspec_workspace_bytes(const ssb_melspec_t* m, const int32_t* sample_offsets, int32_t B);
int ssb_melspec_forward(const ssb_melspec_t* m, const float* wav, const int32_t* sample_offsets, int32_t B, float* mel_out,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ---- vocoder output denoiser --------------------------------------------------------------------------------------------
 * Replaces denoise(wav, v) of tasks/tts/vocoder_infer/hifigan_nsf.py:14-22, which HifiGAN.spec2wav (:73-74) applies to the
 * generator's waveform when hparams['vocoder_denoise_c'] > 0 (same code: vocoders/vocoder_utils.py:7-15): librosa.stft
 * (center=True, pad_mode="constant", periodic Hann window) -> S * max(0, 1 - v / |S|) (= max(|S| - v, 0) e^{i angle S}, 0
 * where |S| = 0) -> librosa.istft (center=True: irfft, window, overlap-add, division by the window sum-square where it exceeds
 * tiny(float32), n_fft / 2 trimmed from each end).  Every utterance is denoised on its own (the reference's B = 1).
 * create: fft_size even, hop_size a multiple of 16, win_length <= fft_size, fft_size <= 32 hop_size (egs/stylesinger.yaml:
 * 1024 / 256 / 1024).  Refused before any CUDA call: bad geometry (create leaves *out NULL), an utterance length that is not
 * a positive multiple of hop_size (the only lengths the vocoder produces; workspace_bytes then returns 0), v < 0 or not
 * finite.  v = 0 is the STFT round trip.  wav_in / wav_out: device fp32 [sum n_b], utterances concatenated, sample_offsets:
 * host [B+1]; the output has the input's length and wav_out may alias wav_in.  Batches of >= 8 row tiles of 128 frames run
 * both DFT GEMMs on the tensor-core kernel (fp16 hi/lo split, 3 MMAs), smaller ones on the fp32 FFMA kernel. */
int ssb_wav_denoise_create(ssb_wav_denoise_t** out, int32_t fft_size, int32_t hop_size, int32_t win_length); /* hifigan_nsf.py:14-22 */
void ssb_wav_denoise_free(ssb_wav_denoise_t* d); /* hifigan_nsf.py:14-22 */
size_t ssb_wav_denoise_workspace_bytes(const ssb_wav_denoise_t* d, const int32_t* sample_offsets, int32_t B); /* hifigan_nsf.py:14-22 */
int ssb_wav_denoise_forward(const ssb_wav_denoise_t* d, const float* wav_in, const int32_t* sample_offsets, int32_t B, float v,
                            float* wav_out, void* workspace, size_t workspace_bytes, void* stream); /* hifigan_nsf.py:14-22 */
/* Test / measurement switch of the GEMM path (hifigan_nsf.py:14-22): 1 = tensor cores on batches of >= 8 row tiles, FFMA
 * below (the default when the tensor-core path is available), 0 = fp32 FFMA always, 2 = tensor cores at every size.
 * Returns the mode in effect (0 when the tensor-core path is unavailable). */
int ssb_wav_denoise_set_tensor_cores(ssb_wav_denoise_t* d, int32_t enable);

/* ---- f3: LSTM utterance encoder of the reference audio (SURVEY.md section 8f) -------------------------------------------
 * Replaces data_gen/tts/emotion/model.py:10-77 (EmotionEncoder: batch-first torch.nn.LSTM 40 -> 256 x 3 layers from zero
 * state + linear 256 -> 256) and the aggregation of data_gen/tts/emotion/inference.py:43-55 (embed_frames_batch) and
 * :150-151 (embed_utterance: mean of the partial embeddings, L2-normalised), which produce the `emo_embed` input of
 * inference/StyleSinger.py:106.  create: HOST fp32 pointers in torch state_dict layout, one per layer -
 * weight_ih[l] [4H, input_size or H], weight_hh[l] [4H, H], bias_ih[l] / bias_hh[l] [4H], gate rows i | f | g | o;
 * linear_weight [embed_size, H] / linear_bias [embed_size] may both be NULL (no `forward` head).  hidden_size must be 256.
 * forward: frames device fp32 [n_partials, n_frames, input_size] (every partial the same length, as the reference batches
 * them).  Outputs (device fp32, each may be NULL, at least one not): hidden_out [n_partials, H] = EmotionEncoder.inference
 * (hidden[-1]); embeds_out [n_partials, embed_size] = EmotionEncoder.forward; utt_embed_out [n_utterances, H] = normalised
 * mean of hidden over partials utt_offsets[u] .. utt_offsets[u+1] (host int32 [n_utterances + 1], 0 .. n_partials, every
 * utterance non-empty; only read when utt_embed_out is given). */
int ssb_lstm_encoder_create(ssb_lstm_encoder_t** out, int32_t input_size, int32_t hidden_size, int32_t num_layers,
                            const float* const* weight_ih, const float* const* weight_hh, const float* const* bias_ih,
                            const float* const* bias_hh, int32_t embed_size, const float* linear_weight, const float* linear_bias);
void ssb_lstm_encoder_free(ssb_lstm_encoder_t* m);
size_t ssb_lstm_encoder_workspace_bytes(const ssb_lstm_encoder_t* m, int32_t n_partials, int32_t n_frames, int32_t n_utterances);
int ssb_lstm_encoder_forward(const ssb_lstm_encoder_t* m, const float* frames, int32_t n_partials, int32_t n_frames,
                             const int32_t* utt_offsets, int32_t n_utterances, float* hidden_out, float* embeds_out,
                             float* utt_embed_out, void* workspace, size_t workspace_bytes, void* stream);

/* Number of kernels this library has launched in this process so far (bench.py reports the delta). */
int64_t ssb_launch_count(void);

/* Diagnostics of the tensor-core GEMM dispatcher (csrc/conv_gemm_tc.cu): launches of one kernel variant, named
 * "tc<BN,MODE>" (single CTA) or "tc2<HB,MODE>" (CTA pair), MODE in GATE / RES_SKIP / GENERIC, e.g. "tc2<64,GENERIC>";
 * the ';'-separated list of variants launched so far (returns their number); and the counters of the activation
 * TMA-descriptor cache (descriptors encoded / served from the cache).  Tests use these to assert WHICH kernel a problem
 * size took; nothing in the reference corresponds to them. */
int64_t ssb_variant_launch_count(const char* variant);
int32_t ssb_variant_names(char* buf, int32_t cap);
void ssb_tensor_map_cache_stats(int64_t* encodes, int64_t* hits);

/* Process-wide switch of the wgmma / TMA attention kernel (csrc/attention_tc.cu) for the long-batch paths of the FFT blocks
 * (common_layers.py:277-286) and of the style aligner's cross-attention (lse.py:41); short batches always use the fp32
 * kernel.  Returns the new state. */
int32_t ssb_set_attention_tensor_cores(int32_t enable);
/* Launches so far of the fp32 attention kernel (tc = 0, csrc/attention.cu) or of the wgmma attention kernel (tc = 1,
 * csrc/attention_tc.cu); any other tc returns 0.  Kept apart from ssb_variant_names, which lists GEMM variants only. */
int64_t ssb_attention_launch_count(int32_t tc);

/* Unit-test granularity: exactly ONE dense GEMM - the fp32 FFMA kernel (path 0, csrc/conv_gemm.cu) or the tensor-core
 * kernel (path 1, csrc/conv_gemm_tc.cu) - with any epilogue, over CALLER-OWNED device buffers in the guard-banded layout
 * of frame_offsets: utterance b occupies rows [rs_b, rs_b + L_b), rs_0 = 16, rs_{b+1} = rs_b + L_b + 16, and `rows` must
 * be rs_{B-1} + L_{B-1} + 16 + 256 (tail slack).  Nothing is copied in or out: buffers may alias (RES_SKIP rewriting its
 * own residual planes, accumulation into `out`), and guard rows, tail slack, column-block-major `out` (out_nb) and the
 * chunk-tiled skip accumulator (skip_tiled) are seen as stored.  Weights are HOST fp32 [N, Cin, k] + bias [N] (may be
 * NULL) in torch layout, packed on the fly (gate != 0: the DiffNet gate interleave, column 2j = sigmoid half j, 2j+1 = tanh
 * half j).  The A operand is fp32 rows [rows, lda] (path 0, with a_act / a_slope / a_scale applied on load) or fp16 hi/lo
 * planes [rows, Cin] (path 1).  The epilogue fields are those of Epi (path 0) and EpiTC (path 1), passed through as they
 * are; the kernels' own checks apply.  Refused before any launch: a conv reach (k - 1) / 2 * dilation beyond the 16 guard
 * rows. */
typedef struct ssb_op_gemm_args {
  int32_t path;                 /* 0: fp32 FFMA, 1: tensor cores */
  const int32_t* frame_offsets; /* host [B + 1] */
  int32_t B;
  int64_t rows;
  int32_t Cin, N, k, dilation, gate;
  const float* w_host;
  const float* b_host;
  const float* a;               /* path 0 */
  int32_t lda, a_act;
  float a_slope, a_scale;
  const void* a_hi;             /* path 1: fp16 [rows, Cin] */
  const void* a_lo;
  int32_t mode;                 /* 0 GENERIC, 1 GATE, 2 RES_SKIP */
  const float* add;
  int32_t ld_add;
  float alpha;
  int32_t act;
  float act_slope;
  const float* res;
  int32_t ld_res;
  float beta;
  const float* rowmask;
  float* out;
  int32_t ldo, accum;
  float gamma;
  float* out2;                  /* path 0 */
  int32_t ldo2;
  const float* vec1;            /* path 1, RES_SKIP with rh / rl */
  const float* vec2;
  void* oh;                     /* fp16 planes: out2_h / out2_l (path 0), oh / ol (path 1) */
  void* ol;
  int32_t ldh, plane_act;
  float plane_slope;
  float* skip;
  int32_t ld_skip, C, skip_init;
  const void* rh;               /* path 1 */
  const void* rl;
  int32_t ld_rh, skip_tiled, out_nb;
  int64_t out_bs;
  void* sh;
  void* sl;
  int32_t n_valid;
  int32_t single_pass;          /* path 1 only: 0 = the 3-pass fp16 hi/lo split (a_lo read), 1 = one hi*hi pass (a_lo unread,
                                   may be NULL) - the kernel of SSB_TC_FP16.  Anything else, or 1 on path 0, is refused. */
} ssb_op_gemm_args;
int ssb_op_gemm(const ssb_op_gemm_args* a, void* stream);
/* Unit-test granularity: exactly ONE attention call - the fp32 kernel (path 0, csrc/attention.cu) or the wgmma kernel
 * (path 1, csrc/attention_tc.cu) - over CALLER-OWNED device buffers in the guard-banded layouts of q_offsets (queries,
 * rows_q rows) and k_offsets (keys and values, rows_k rows): utterance b at rows [rs_b, rs_b + L_b), rs_0 = 16,
 * rs_{b+1} = rs_b + L_b + 16, and rows_* must be rs_{B-1} + L_{B-1} + 16 + 256 (tail slack).  Query utterance b attends to
 * key utterance b; head h (of `heads`, 128 columns each) reads columns 128 h of each operand's window.  Nothing is copied
 * in or out; rows outside the utterances are never written.
 *   path 0: q / k / v fp32 [rows, ld*] (column windows by pointer offset, as the FFT blocks pass qkv + 256); output fp32
 *           out [rows_q, ldo] only; qcol0 / kcol0 / vcol0 must be 0.
 *   path 1: q_hi / q_lo, k_hi / k_lo, v_hi / v_lo fp16 planes [rows, ld*] with the window at column *col0; V's planes are
 *           transposed into the call's own V^T scratch (ldvt = (rows_k + 7) & ~7) first, as the stage drivers do (one
 *           transpose_planes launch).  Output fp32 out [rows_q, ldo], fp16 planes oh / ol [rows_q, ldh], or both.
 * keymask: optional guarded device [rows_k], 0 = masked key.  An utterance with no valid key gets NaN rows.
 * Refused before any launch: a path other than 0 / 1; no output, or a plane output on path 0; fp32 lds not multiples of 4
 * or fp32 pointers not 16-byte aligned; path 1 lds or column offsets not multiples of 8, or planes not 16-byte aligned; a
 * column window past its ld; heads outside {1, 2}; rows_q / rows_k that do not match their layout; B > 65535.  The stage
 * drivers' attention calls make the same checks. */
typedef struct ssb_op_attention_args {
  int32_t path;                 /* 0: fp32 kernel, 1: wgmma kernel */
  const int32_t* q_offsets;     /* host [B + 1] */
  const int32_t* k_offsets;     /* host [B + 1] */
  int32_t B;
  int64_t rows_q, rows_k;
  int32_t heads;
  float scale;                  /* applied to q */
  const float* keymask;
  const float* q;               /* path 0 */
  const float* k;
  const float* v;
  const void* q_hi;             /* path 1 */
  const void* q_lo;
  const void* k_hi;
  const void* k_lo;
  const void* v_hi;
  const void* v_lo;
  int32_t ldq, qcol0, ldk, kcol0, ldv, vcol0;
  float* out;
  int32_t ldo;
  void* oh;                     /* path 1 */
  void* ol;
  int32_t ldh;
} ssb_op_attention_args;
int ssb_op_attention_ex(const ssb_op_attention_args* a, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STYLESINGER_B200_H */
