#pragma once
#include "model.cuh"

namespace ssb {

int fft_blocks(Ctx& c, const FFT& f, const SeqDev& s, float* x, const float* keep, bool tc = false);
int run_encoder(Ctx& c, const Model& m, const SeqDev& sp, const int32_t* tok_g, const int32_t* note_g,
                const int32_t* type_g, const float* ndur_g, float* srcmask, float* enc_out);
int run_fft_decoder(Ctx& c, const Model& m, const SeqDev& sf, const float* dec_in, float* xd, bool tc);
int run_duration_predictor(Ctx& c, const Model& m, const SeqDev& sp, const float* dur_inp, const float* srcmask,
                           float* logdur, int32_t* dur);
// f0_gen 'conv': one PitchPredictor (which 0: pitch_predictor, 1: pitch_inpainter_predictor), x [rows,256] -> out
// [rows,2]; tc: the five convs on the tensor-core kernel
int run_pitch_predictor(Ctx& c, const Model& m, int which, const SeqDev& s, const float* x_g, float* out_g, bool tc);
int run_style(Ctx& c, const Model& m, const SeqDev& sf, const SeqDev& sr, const float* dec0, const float* ref_g,
              const float* reff0_g, float* style, int32_t* codes, float* rq_in_out);
struct DenoiserBufs {
  float *x, *y, *zg, *skip, *sbuf, *head, *condall;
  float* condpre;             // tensor-core path: hoisted conditioner projection, [rows, 2C] fp32 pre-activation addends per layer
  __half *yh, *yl, *zh, *zl;  // tensor-core path: fp16 hi/lo planes of y = x + step bias and of the gate output
  __half *ch, *cl;            // tensor-core path: fp16 hi/lo planes of the conditioner [rows,256] (A of the hoisted projection)
  __half *skh, *skl, *sh, *sl;  // tensor-core heads: planes of the skip sum and of relu(skip_proj)
  __half *x80h, *x80l;          // mel net, tensor-core in_proj: planes of x_t padded to 128 columns
  bool tc_heads;                // also: the skip accumulator is in the chunk-tiled layout (EpiTC::skip_tiled)
  int ld_head;
  bool tc;
};
bool denoiser_tc_ok(const Model& m, const Denoiser& d);
int alloc_denoiser(Ctx& c, const Denoiser& d, const SeqDev& s, bool tc, DenoiserBufs* b);
int prepare_cond(Ctx& c, const Denoiser& d, const SeqDev& s, const float* cond_g, DenoiserBufs& b);
int mel_denoiser_eval(Ctx& c, const Denoiser& d, const SeqDev& s, int t, const float* x80, DenoiserBufs& b);
int denoiser_stack(Ctx& c, const Denoiser& d, const SeqDev& s, int t, DenoiserBufs& b);
// host_seq (optional): the host-side layout of `s`; needed for the utterance grouping of ssb_model_set_persistent_groups
int run_mel_diffusion(Ctx& c, const Model& m, const SeqDev& s, const float* cond_g, const float* coarse_g,
                      const float* noise, uint64_t seed, float* mel_tight, const Seq* host_seq = nullptr);
int run_mel_diffusion_plms(Ctx& c, const Model& m, const SeqDev& s, const float* cond_g, const float* coarse_g,
                           const float* q_noise, uint64_t seed, int interval, float* mel_tight);
int run_f0_diffusion(Ctx& c, const Model& m, int which, const SeqDev& s, const float* cond_g, const float* lo,
                     const float* hi, const float* gnoise, const float* unoise, uint64_t seed, float* z, int32_t* uv);
// both F0 samplers (agnostic: cond0, gnoise[0], ... ; specific: cond1, gnoise[1], ...)
int run_f0_samplers(Ctx& c, const Model& m, const SeqDev& s, const float* cond0, const float* cond1, const float* lo,
                    const float* hi, const float* const gnoise[2], const float* const unoise[2], uint64_t seed,
                    float* const z[2], int32_t* const uv[2]);
int run_vocoder(Ctx& c, const Vocoder& v, const Seq& seq, const float* mel_tight, const float* f0_tight,
                const float* rand_ini, const float* src_noise, uint64_t seed, float* wav_tight);
int denoiser_eval_api(Ctx& c, const Model& m, int which, const SeqDev& s, const float* x_tight, const int32_t* uv_tight,
                      int t, const float* cond_tight, float* out_tight);
int run_acoustic(Ctx& c, const Model& m, const ssb_acoustic_inputs& in, const ssb_acoustic_outputs& out, bool durations_only,
                 int32_t* dur_out, float* logdur_out);

}  // namespace ssb
