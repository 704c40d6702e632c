// Packed (device-resident) weights of the acoustic model and the vocoder, plus the stage drivers.
#pragma once
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/stylesinger_b200.h"
#include "attention.cuh"
#include "common.cuh"
#include "conv_gemm.cuh"
#include "conv_gemm_tc.cuh"
#include "ops.cuh"

namespace ssb {

// One dense operator: weights [taps][Cin][Npad] + bias [N]
struct Conv {
  float* W = nullptr;
  float* bias = nullptr;
  int taps = 1, Cin = 0, N = 0, Npad = 0, dil = 1, center = 0;
};

// A dense layer whose weights are packed for both GEMMs: fp32 FFMA (conv_gemm) and tensor cores (conv_gemm_tc; t.ok is
// false when the shape is not eligible).  run_dense (stages.cuh) enqueues either.
struct Dense {
  Conv f;
  ConvTC t;
};

enum PackMode { PACK_PLAIN = 0, PACK_GATE_SIG_TANH = 1 /* DiffNet: [sigmoid C | tanh C] */,
                PACK_GATE_TANH_SIG = 2 /* WN: [tanh C | sigmoid C] */ };

struct HostTensor {
  const float* data = nullptr;
  std::vector<int64_t> shape;
  int64_t numel() const {
    int64_t n = 1;
    for (auto s : shape) n *= s;
    return n;
  }
};

// Owns every cudaMalloc'ed weight buffer.
struct DevicePool {
  std::vector<void*> ptrs;
  ~DevicePool();
  float* upload(const std::vector<float>& h);
  float* alloc(size_t n);
  void release(void* p);  // free one buffer of the pool early (schedule tables replaced by ssb_model_set_schedule)
};

struct TensorMap {
  std::map<std::string, HostTensor> t;
  std::string missing;
  const HostTensor* get(const std::string& name, std::initializer_list<int64_t> shape = {});
};

struct FFTLayer {
  float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  // the FFN is 92 % of the block's FLOPs; the tensor-core packing of all four is used for long sequences
  Dense qkv, out, ffn1, ffn2;
};
struct FFT {
  std::vector<FFTLayer> layers;
  bool tc_ok = true;  // every layer's four GEMMs are tensor-core eligible
  float *ln_g = nullptr, *ln_b = nullptr;
  float* pos_alpha = nullptr;  // device scalar, null for the encoder
  int kernel = 9;
};

struct DenoiserLayer {
  Dense dil;   // k3 dilated, gate-interleaved columns, N = 2C
  Dense outp;  // 1x1, N = 2C ([res | skip])
  Conv dproj;  // diffusion_projection C -> C (used only to build the step-bias table)
  float* bias_gate_tc = nullptr;  // dil bias + conditioner bias (packed column order): the GATE GEMM's bias (cond_all_tc has none)
};
struct Denoiser {
  int C = 0, L = 0, in_dims = 0, out_dims = 0, cycle = 4;
  bool ddiff = false;
  Conv in_proj;                 // mel: 80 -> C (relu).  ddiff: unused (in_w / in_b below)
  float *in_w = nullptr, *in_b = nullptr, *uv_emb = nullptr;  // ddiff input: [C/2], [C/2], [2][C/2]
  Conv mlp0, mlp2;
  std::vector<DenoiserLayer> layers;
  Conv cond_all;                // 256 -> L*2C, gate-interleaved per layer
  ConvTC cond_all_tc;           // the same stacked projection for the tensor-core kernel (hoisted out of the T loop; no bias)
  bool tc_ok = false;           // cond_all_tc and every layer's dil / outp are tensor-core eligible
  Conv skip_proj, out_proj;
  // schedule-dependent (set by ssb_model_set_schedule)
  int T = 0;
  float* dtab = nullptr;        // [T][L][C] step bias per layer
  float* gtab = nullptr;        // [T][8]
  float* mtab = nullptr;        // [T][8] (ddiff only)
  std::vector<float> gtab_h;
  // persistent-sampler extras (mel net): every GEMM of a diffusion step on the tensor-core path
  ConvTC in_tc;    // input_projection, K padded 80 -> 128
  ConvTC skip_tc;  // skip_projection with the 1/sqrt(L) skip scale folded into the weights
  ConvTC out_tc;   // output_projection, N padded 80 -> 256 (4 N-tiles of 64: one cluster)
  float* out_bias_pad = nullptr;
  float* skip_bias_pad = nullptr;
};

// FastSpeech-2 PitchPredictor (tts_modules.py:191-234): f0_gen 'conv' only
struct PitchPredictor {
  static constexpr int kLayers = 5;
  Dense conv[kLayers];      // k-tap Conv1d 256 -> 256 + bias; the tensor-core packing is used for long batches
  bool tc_ok = true;        // all of them are tensor-core eligible
  float* ln_g[kLayers] = {};
  float* ln_b[kLayers] = {};
  Conv linear;              // 256 -> 2
  float* pos_alpha = nullptr;  // device scalar
};

struct AlignLayer {
  Dense q, kv, out, lin1, lin2;  // the tensor-core packing is used for long batches
  float *n1_g, *n1_b, *n2_g, *n2_b;
};

struct Model {
  DevicePool pool;
  ssb_hparams hp;
  // tables
  float* pos_table = nullptr; int pos_rows = 0;
  float* tok_emb = nullptr; int n_tokens = 0;
  float *note_emb = nullptr, *type_emb = nullptr, *dur_w = nullptr, *dur_b = nullptr;
  float* pitch_emb = nullptr;
  float *spec_min = nullptr, *spec_max = nullptr;
  Conv spk_proj, emo_proj;
  // hparams['use_spk_id'] (ssb_model_create_ex4): spk_embed_proj is an Embedding [spk_rows, 256] looked up by the host's
  // speaker ids instead of the Linear spk_proj over a speaker vector
  bool spk_id = false;
  float* spk_tab = nullptr;
  int spk_rows = 0;
  FFT enc, dec;
  Conv dp_conv[4]; float* dp_ln_g[4]; float* dp_ln_b[4]; Conv dp_lin; int dp_layers = 2;
  // style adaptor
  Conv wn_in[4], wn_rs[4];
  struct CB { float *ln_g, *ln_b; Conv c1, c2; } cb[10];
  float *cb_last_g = nullptr, *cb_last_b = nullptr;
  Conv cb_post;
  float* codebooks = nullptr; float* cb_norm2 = nullptr;  // [depth][n_embed][256], [depth][n_embed]
  Conv l1;
  AlignLayer align[2];
  bool align_tc_ok = true;  // all ten projections are tensor-core eligible
  Denoiser f0net[2];        // GMDIFF only
  PitchPredictor pp[2];     // CONV only: [0] pitch_predictor (domain agnostic), [1] pitch_inpainter_predictor (specific)
  // SSB_F0_GEN_GMDIFF: hparams['f0_gen'] == 'gmdiff' (two F0 diffusion samplers); SSB_F0_GEN_CONV: 'conv' (pp above)
  int f0_gen = SSB_F0_GEN_GMDIFF;
  Denoiser melnet;
  Conv mel_out, ln_proj;  // mel_out: DiffSinger and FFT modes; ln_proj: DiffSinger mode only
  // SSB_MEL_DECODER_DIFFSINGER: hparams['decoder'] == 'diffsinger' (FFT decoder + mel_out + ln_proj + DDPM over postdiff.*);
  // SSB_MEL_DECODER_PRODIFF: 'prodiff' (decoder_inp straight into the x0-predicting sampler over diff_decoder.*);
  // SSB_MEL_DECODER_FFT: 'fft' (FFT decoder + mel_out is the mel; no melnet)
  int mel_decoder = SSB_MEL_DECODER_DIFFSINGER;
  // model switches (ssb_model_create_ex3): emo_proj is packed only with emo; the style adaptor, codebooks, l1 and align only
  // with style; umln builds nothing (identity at inference); use_txt_cond adds decoder_inp to ln_proj's input
  ssb_model_switches sw = {1, 1, 1, 1};
  int cond_width = 1104;  // ln_proj's input width: 80 + 256 (1 + use_txt_cond + emo + style)
  // hparams['K_step'] of the DiffSinger mel sampler (ssb_model_set_mel_k_step): q_sample at K-1, then K reverse steps on the
  // T-step schedule.  0 follows the schedule's T.
  int mel_k_step = 0;
  float log_eps = 0.f;
  // auxiliary stream + fork/join events: lets the two independent F0 samplers overlap (created in build_model).
  // Calls on one model are therefore serialised with respect to these events (one in-flight forward per model).
  cudaStream_t aux_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  bool persistent = true;  // single-launch persistent sampler for small batches (ssb_model_set_persistent)
  bool persistent_groups = false;  // large batches: groups of <= 48 row tiles, one persistent launch each (mel sampler)
  bool use_tc = true;  // tensor-core path for the denoiser layer GEMMs (ssb_model_set_tensor_cores)
  bool fft_tc = true;  // tensor-core path for the decoder FFT blocks' FFN on long batches (ssb_model_set_fft_tensor_cores)
  // SSB_TC_FP16 (ssb_model_set_mel_precision): the mel DiffNet's tensor-core GEMMs run single-pass fp16 (GemmTC::single_pass)
  bool mel_fp16 = false;
};

struct VocStage {
  Dense up;         // transposed conv as 3-tap conv, N = u * Cout
  int u = 1, Cout = 0;
  float *nc_w = nullptr, *nc_b = nullptr; int nc_s = 1;  // noise conv
  float* nc_wt = nullptr;                                 // the same weights as [K, C] (tiled kernel)
  // ResBlock1: convs1.{m} / convs2.{m} in c1[m] / c2[m]; ResBlock2: convs.{m} in c1[m] (c2 unused).  A grouped stage
  // (g > 1) holds the grouped packing in the tensor-core halves, and at C < 32 in the FFMA halves as well.
  struct RB { Dense c1[3], c2[3]; } rb[4];
  bool res_tc = false;  // all ResBlock convs of this stage have a tensor-core packing (C % 64 == 0, or grouped)
  // time-group factor 64 / C (C = 32, 16, 8): the ResBlock convs are packed as 64-channel convs over groups of g
  // consecutive time steps, i.e. over the [rows/g, 64] view of the [rows, C] buffers (see pack.cu); 1: not grouped
  int g = 1;
};
struct Vocoder {
  DevicePool pool;
  ssb_vocoder_config_ex cfg;
  Conv pre, post;
  std::vector<VocStage> stages;
  int nk = 3;
  int resblock = 1;  // 1: ResBlock1 (3 conv pairs per block), 2: ResBlock2 (2 single convs per block)
  float *lin_w = nullptr, *lin_b = nullptr;
  bool nsf = true;
  bool use_tc = true;
  bool fp16 = false;  // SSB_TC_FP16 (ssb_vocoder_set_precision): tensor-core GEMMs single-pass fp16
};

// ---- packing helpers (pack.cu) -------------------------------------------------------------------
int pack_conv(DevicePool& pool, const HostTensor* w, const HostTensor* b, int dil, PackMode mode, Conv* out,
              const HostTensor* g = nullptr /* weight-norm g: w is v */);
int pack_conv_tc(DevicePool& pool, const HostTensor* w, int dil, PackMode mode, const float* packed_bias, ConvTC* out);
int pack_linear(DevicePool& pool, const HostTensor* w, const HostTensor* b, Conv* out);
// both packings of one layer from one tensor: w [N, Cin, k], or a Linear's [N, Cin] as a 1-tap conv, rows [row0, row0 + nrows)
int pack_dense(DevicePool& pool, const HostTensor* w, const HostTensor* b, int dil, PackMode mode, Dense* out,
               const HostTensor* g = nullptr /* weight-norm g: w is v */, int row0 = 0, int nrows = -1);
int pack_conv_transpose(DevicePool& pool, const HostTensor* v, const HostTensor* g, const HostTensor* b, int u, Conv* out);
int build_model(TensorMap& tm, const ssb_hparams& hp, Model* m, int mel_decoder, int f0_gen, const ssb_model_switches& sw,
                bool use_spk_id);
// ln_proj's input width under the switches sw (stylesinger.py:92-100)
inline int cond_width(const ssb_model_switches& sw) { return 80 + 256 * (1 + sw.use_txt_cond + sw.emo + sw.style); }
int build_vocoder(TensorMap& tm, const ssb_vocoder_config_ex& cfg, Vocoder* v);
int set_schedule(Model* m, int which, int T, const float* step_emb, const float* gtab, const float* mtab,
                 cudaStream_t stream);

// ---- op helpers (stages.cu) ------------------------------------------------------------------------
ConvGemm make_gemm(const Conv& c, const SeqDev& s, const float* A, int lda);
GemmTC make_gemm_tc(const ConvTC& w, const SeqDev& s, const __half* A_hi, const __half* A_lo);

}  // namespace ssb
