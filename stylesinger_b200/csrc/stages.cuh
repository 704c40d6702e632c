#pragma once
#include "model.cuh"

namespace ssb {

#define RUN(x)                 \
  do {                         \
    int rc_ = (x);             \
    if (rc_ != 0) return rc_;  \
  } while (0)
#define WS_OK(c) SSB_CHECK((c).dry || !(c).failed, "workspace too small")

// zero-filled guard-banded rows of other element types (alloc_rows: common.cuh)
int32_t* alloc_rows_i32(Ctx& c, const SeqDev& s, int C = 1);
__half* alloc_half_rows(Ctx& c, const SeqDev& s, int C);

// Long batches (>= 8 row tiles) run the FFT decoder, the aligner and the pitch predictors on the tensor-core kernel
bool long_batch_tc(const Model& m, const SeqDev& s);

// The input act(x) of a dense layer: fp32 rows x (the FFMA kernel applies act on load) and / or fp16 hi/lo planes that
// already hold act(x) (written by the producing epilogue or by split_planes).  A path reads the form it needs.
struct DenseIn {
  const float* x = nullptr;
  int ld = 0;
  const __half *hi = nullptr, *lo = nullptr;
  int act = ACT_NONE;  // ACT_NONE or ACT_LRELU
  float slope = 0.1f;
};
// Enqueues the layer over the rows of `s` on the tensor-core (tc) or the fp32 FFMA kernel.  `e` describes the epilogue
// for both (bias: the layer's own); a field the chosen kernel cannot honour is an error.  single_pass: the tensor-core
// kernel's single-pass fp16 mode (GemmTC::single_pass); the FFMA kernel ignores it.
int run_dense(Ctx& c, const Dense& d, bool tc, const SeqDev& s, const DenseIn& in, const Epi& e, bool single_pass = false);

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
  bool single_pass;             // tensor-core path: single-pass fp16 GEMMs (the mel net under SSB_TC_FP16); false from alloc_denoiser
};
bool denoiser_tc_ok(const Model& m, const Denoiser& d);
int alloc_denoiser(Ctx& c, const Denoiser& d, const SeqDev& s, bool tc, DenoiserBufs* b);
int prepare_cond(Ctx& c, const Denoiser& d, const SeqDev& s, const float* cond_g, DenoiserBufs& b);
int mel_denoiser_eval(Ctx& c, const Denoiser& d, const SeqDev& s, int t, const float* x80, DenoiserBufs& b);
int denoiser_stack(Ctx& c, const Denoiser& d, const SeqDev& s, int t, DenoiserBufs& b);
// The samplers' Philox draws are keyed by the layout's table (SeqDev::rng, from Seq::seed / Seq::utt_seeds).
// host_seq (optional): the host-side layout of `s`; needed for the utterance grouping of ssb_model_set_persistent_groups
int run_mel_diffusion(Ctx& c, const Model& m, const SeqDev& s, const float* cond_g, const float* coarse_g,
                      const float* noise, float* mel_tight, const Seq* host_seq = nullptr);
int run_mel_diffusion_plms(Ctx& c, const Model& m, const SeqDev& s, const float* cond_g, const float* coarse_g,
                           const float* q_noise, int interval, float* mel_tight);
int run_f0_diffusion(Ctx& c, const Model& m, int which, const SeqDev& s, const float* cond_g, const float* lo,
                     const float* hi, const float* gnoise, const float* unoise, float* z, int32_t* uv);
// both F0 samplers (agnostic: cond0, gnoise[0], ... ; specific: cond1, gnoise[1], ...)
int run_f0_samplers(Ctx& c, const Model& m, const SeqDev& s, const float* cond0, const float* cond1, const float* lo,
                    const float* hi, const float* const gnoise[2], const float* const unoise[2], float* const z[2],
                    int32_t* const uv[2]);
// seq.seed / seq.utt_seeds key the NSF source's draws
int run_vocoder(Ctx& c, const Vocoder& v, const Seq& seq, const float* mel_tight, const float* f0_tight,
                const float* rand_ini, const float* src_noise, float* wav_tight);
int denoiser_eval_api(Ctx& c, const Model& m, int which, const SeqDev& s, const float* x_tight, const int32_t* uv_tight,
                      int t, const float* cond_tight, float* out_tight);
// ---- implicit-GEMM STFT pieces shared by the mel front-end and the vocoder output denoiser (frontend.cu) ----------------
// A frame of n_fft samples centred on sample t * hop is `span / hop` consecutive rows of hop samples (rows t - taps/2 ..
// t + taps/2 - 1), span = n_fft rounded up to a multiple of 2 hop, with (span - n_fft) / 2 zero-weight samples on each side.
int stft_span(int n_fft, int hop);
// librosa.stft, center=True: 1 + n / hop frames; the frame layout of a batch of waveforms (sample_offsets: host [B+1])
int frames_of(int64_t n, int hop);
int build_seq(const int32_t* sample_offsets, int B, int hop, Seq* q);
// tight waveform -> rows of hop samples in the frame layout `s` (zero behind the last sample); sample_offs_dev: device [B+1]
int wav_rows(Ctx& c, const SeqDev& s, const int32_t* sample_offs_dev, const float* wav, int hop, float* rows);
// periodic Hann window of `win` samples zero-padded (centred) to n_fft, float64 (librosa's 'hann' window)
std::vector<double> hann_window(int n_fft, int win);
// windowed DFT basis of one frame, [span][2 nbp] = (re | im) columns of bins 0 .. n_fft/2 (padding columns zero); row i is
// frame sample i - lead.  inverse = false: w[j] cos, -w[j] sin (rfft of the windowed frame, librosa.stft).  inverse = true:
// c_k w[j] cos, -c_k w[j] sin with c_k = 1 for bins 0 and n_fft/2 (whose imaginary parts numpy's irfft ignores: zero) and
// 2 otherwise, i.e. irfft times the window of librosa.istft WITHOUT its 1/n_fft (the caller scales the GEMM's output).
std::vector<float> dft_basis(int n_fft, int hop, int win, int nbp, bool inverse);

// utt_seeds (host [B] or null): per-utterance Philox keys of the samplers; null keys them all by in.seed
int run_acoustic(Ctx& c, const Model& m, const ssb_acoustic_inputs& in, const ssb_acoustic_outputs& out, bool durations_only,
                 int32_t* dur_out, float* logdur_out, const uint64_t* utt_seeds = nullptr);

}  // namespace ssb
