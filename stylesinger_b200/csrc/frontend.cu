// f3 (SURVEY.md section 8f): the mel-spectrogram half of the reference-audio front-end.
//   librosa_wav2spec (reference utils/audios/__init__.py:36-84, called from inference/StyleSinger.py:79-92):
//     x_stft = librosa.stft(wav, n_fft, hop_length, win_length, window="hann", pad_mode="constant")   (center=True)
//     mel    = log10(max(eps, mel_basis @ |x_stft|)),  mel_basis = librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)
// As kernels: the waveform of every utterance is laid out as rows of `hop` samples in the guard-banded ragged layout, so a
// frame (n_fft = taps * hop samples centred on sample t * hop) is `taps` consecutive rows and the windowed real DFT is ONE
// implicit-GEMM conv over those rows (conv_gemm: taps = n_fft / hop, Cin = hop, N = 2 * bins, weights = window x cos / -sin);
// the zero guard rows ARE librosa's centre padding.  Then |.| , the mel filterbank as a second GEMM, log10(max(eps, .)).
// fp32 FFMA throughout (4.3 MFLOP per frame: nothing here is worth a tensor core).  The speaker / emotion encoders and the
// Praat pitch tracker of the reference's preprocess_input are NOT part of this file (third-party models, see DESIGN.md).
#include <math.h>

#include <algorithm>
#include <memory>
#include <vector>

#include "../../include/stylesinger_b200.h"
#include "conv_gemm.cuh"
#include "model.cuh"
#include "stages.cuh"

struct ssb_melspec {
  ssb::DevicePool pool;
  ssb::Conv dft;   // [taps][hop][2 * nbp]  (re | im), window folded in
  ssb::Conv mel;   // [1][nbp][n_mels]
  int sample_rate = 0, n_fft = 0, hop = 0, win = 0, n_mels = 0, nbins = 0, nbp = 0, taps = 0;
  float eps = 1e-6f;
  int reflect = 0;  // centre padding: 0 = zeros (librosa_wav2spec passes pad_mode="constant"), 1 = np.pad "reflect" (librosa default)
  int power = 0;    // 0 = |X| (librosa_wav2spec), 1 = |X|^2 (librosa.feature.melspectrogram default power=2.0)
  int log10 = 1;    // 1 = log10(max(eps, mel)), 0 = the filterbank output itself
};

namespace ssb {

ConvGemm make_gemm(const Conv& c, const SeqDev& s, const float* A, int lda);  // stages.cu

// tight waveform [sum n_b] -> rows of `hop` samples in the guard-banded layout (zero fill behind the last sample)
__global__ void k_wav_rows(const int4* utt, const int32_t* sample_offs, const float* wav, int hop, float* rows) {
  const int b = blockIdx.y;
  const int4 u = utt[b];
  const int64_t n = (int64_t)sample_offs[b + 1] - sample_offs[b];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // sample index inside the utterance's row block
  if (i >= (int64_t)u.y * hop) return;
  rows[(int64_t)u.x * hop + i] = i < n ? wav[(int64_t)sample_offs[b] + i] : 0.f;
}

int wav_rows(Ctx& c, const SeqDev& s, const int32_t* sample_offs_dev, const float* wav, int hop, float* rows) {
  if (c.dry || s.B == 0) return 0;
  const int64_t per = (int64_t)s.maxlen * hop;
  k_wav_rows<<<dim3((unsigned)((per + 255) / 256), (unsigned)s.B), 256, 0, c.stream>>>(s.utt, sample_offs_dev, wav, hop, rows);
  SSB_CUDA(cudaGetLastError());
  ++g_launches;
  return 0;
}

int frames_of(int64_t n, int hop) { return (int)(1 + n / hop); }  // librosa.stft, center=True

int build_seq(const int32_t* sample_offsets, int B, int hop, Seq* q) {
  std::vector<int32_t> fo((size_t)B + 1, 0);
  for (int b = 0; b < B; ++b) {
    const int64_t n = (int64_t)sample_offsets[b + 1] - sample_offsets[b];
    SSB_CHECK(n >= 0, "sample offsets must be non-decreasing");
    fo[(size_t)b + 1] = fo[(size_t)b] + frames_of(n, hop);
  }
  q->build(fo.data(), B);
  return 0;
}

int stft_span(int n_fft, int hop) { return (n_fft + 2 * hop - 1) / (2 * hop) * (2 * hop); }

std::vector<double> hann_window(int n_fft, int win) {
  // scipy.signal.get_window("hann", win_length, fftbins=True), zero-padded on both sides to n_fft (librosa.util.pad_center)
  const double PI = 3.14159265358979323846;
  std::vector<double> w((size_t)n_fft, 0.0);
  const int lpad = (n_fft - win) / 2;
  for (int i = 0; i < win; ++i) w[(size_t)lpad + i] = 0.5 - 0.5 * cos(2.0 * PI * i / win);
  return w;
}

std::vector<float> dft_basis(int n_fft, int hop, int win, int nbp, bool inverse) {
  const double PI = 3.14159265358979323846;
  const std::vector<double> w = hann_window(n_fft, win);
  const int span = stft_span(n_fft, hop), lead = (span - n_fft) / 2, nbins = n_fft / 2 + 1, N2 = 2 * nbp;
  std::vector<float> W((size_t)span * N2, 0.f);  // [tap][c][n]: row sample tap * hop + c = frame sample j + lead
  for (int j = 0; j < n_fft; ++j)
    for (int k = 0; k < nbins; ++k) {
      const double ph = 2.0 * PI * (double)(((int64_t)j * k) % n_fft) / n_fft;
      if (!inverse) {
        W[(size_t)(j + lead) * N2 + k] = (float)(w[(size_t)j] * cos(ph));
        W[(size_t)(j + lead) * N2 + nbp + k] = (float)(-w[(size_t)j] * sin(ph));
      } else {
        const bool edge = k == 0 || 2 * k == n_fft;  // numpy's irfft ignores the imaginary parts of the DC and Nyquist bins
        const double ck = edge ? 1.0 : 2.0;
        W[(size_t)(j + lead) * N2 + k] = (float)(ck * w[(size_t)j] * cos(ph));
        W[(size_t)(j + lead) * N2 + nbp + k] = edge ? 0.f : (float)(-ck * w[(size_t)j] * sin(ph));
      }
    }
  return W;
}

namespace {

// np.pad(y, n_fft / 2, mode="reflect") of librosa.stft's default centring.  numpy reflects as often as the pad needs, i.e.
// sample p (p < 0 or p >= n) is the even periodic extension of y with period 2 (n - 1): sample -i is y[i], sample n - 1 + i
// is y[n - 1 - i] while i < n, and a 1-sample clip pads with y[0].  (numpy refuses n == 0; so does run_melspec.)
__device__ __forceinline__ int64_t reflect_src(int64_t p, int64_t n) {
  if (n == 1) return 0;
  const int64_t per = 2 * (n - 1);
  int64_t q = p % per;
  if (q < 0) q += per;
  return q < n ? q : per - q;
}
// Written into the guard rows in front of the utterance and behind its last sample (pad <= 8 rows each side; the 16 guard
// rows between neighbours keep the two utterances' pads apart).
__global__ void k_wav_reflect(const int4* utt, const int32_t* sample_offs, const float* wav, int hop, int pad, float* rows) {
  const int b = blockIdx.y;
  const int4 u = utt[b];
  const int64_t n = (int64_t)sample_offs[b + 1] - sample_offs[b];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // 0 .. 2 pad: [0, pad) = left pad, [pad, 2 pad) = right pad
  if (i >= 2 * pad || n == 0) return;
  const float* y = wav + sample_offs[b];
  if (i < pad) {
    rows[(int64_t)u.x * hop - 1 - i] = y[reflect_src(-1 - (int64_t)i, n)];
  } else {
    const int j = i - pad;
    rows[(int64_t)u.x * hop + n + j] = y[reflect_src(n + j, n)];
  }
}
// |re + i im| for the [rows, 2 * nbp] (re | im) spectrum; columns >= nbins are padding (zero weights -> zero)
__global__ void k_magnitude(const float* spec, int64_t rows, int nbp, int power, float* mag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * nbp) return;
  const int64_t r = i / nbp;
  const int c = (int)(i - r * nbp);
  const float re = spec[r * 2 * nbp + c], im = spec[r * 2 * nbp + nbp + c];
  const float p2 = re * re + im * im;
  mag[i] = power ? p2 : sqrtf(p2);
}
__global__ void k_log10_unpack(const int4* utt, const float* x, int ld, int C, float eps, int take_log, float* out_tight) {
  const int b = blockIdx.y;
  const int4 u = utt[b];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)u.y * C) return;
  const int64_t t = i / C;
  const int c = (int)(i - t * C);
  const float v = x[((int64_t)u.x + t) * ld + c];
  out_tight[((int64_t)u.z + t) * C + c] = take_log ? log10f(fmaxf(eps, v)) : v;
}

// librosa 0.8 filters.mel (Slaney scale, htk=False, norm='slaney'), float64 like numpy, then float32
double hz_to_mel(double f) {
  const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
  return f >= min_log_hz ? min_log_mel + log(f / min_log_hz) / logstep : f / f_sp;
}
double mel_to_hz(double m) {
  const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
  return m >= min_log_mel ? min_log_hz * exp(logstep * (m - min_log_mel)) : f_sp * m;
}

int run_melspec(Ctx& c, const ssb_melspec& m, const Seq& q, const float* wav, const int32_t* sample_offsets_host, int B, float* mel_out) {
  if (m.reflect)  // before any copy or launch, and in the dry run that sizes the workspace
    for (int b = 0; b < B; ++b)
      SSB_CHECK(sample_offsets_host[b + 1] > sample_offsets_host[b], "reflect padding needs at least one sample per utterance (numpy refuses an empty array)");
  SeqDev s;
  RUN(upload_layout(c, q, 1, &s));
  int32_t* offs_dev = c.alloc<int32_t>((size_t)B + 1);
  float* rows = alloc_rows(c, s, m.hop);           // zero-filled incl. guards = centre padding
  float* spec = alloc_rows(c, s, 2 * m.nbp, false);
  float* mag = alloc_rows(c, s, m.nbp, false);
  float* mel = alloc_rows(c, s, m.n_mels, false);
  WS_OK(c);
  if (c.dry || B == 0) return 0;
  SSB_CUDA(cudaMemcpyAsync(offs_dev, sample_offsets_host, sizeof(int32_t) * ((size_t)B + 1), cudaMemcpyHostToDevice, c.stream));
  RUN(wav_rows(c, s, offs_dev, wav, m.hop, rows));
  if (m.reflect) {
    const int pad = m.n_fft / 2;
    k_wav_reflect<<<dim3((unsigned)((2 * pad + 255) / 256), (unsigned)B), 256, 0, c.stream>>>(s.utt, offs_dev, wav, m.hop, pad, rows);
    SSB_CUDA(cudaGetLastError());
    ++g_launches;
  }
  {
    ConvGemm g = make_gemm(m.dft, s, rows, m.hop);
    g.e.out = spec; g.e.ldo = 2 * m.nbp;
    RUN(conv_gemm(c, g));
  }
  {
    const int64_t n = s.rows * m.nbp;
    k_magnitude<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(spec, s.rows, m.nbp, m.power, mag);
    SSB_CUDA(cudaGetLastError());
    ++g_launches;
  }
  {
    ConvGemm g = make_gemm(m.mel, s, mag, m.nbp);
    g.e.out = mel; g.e.ldo = m.n_mels;
    RUN(conv_gemm(c, g));
  }
  {
    const int64_t per = (int64_t)s.maxlen * m.n_mels;
    k_log10_unpack<<<dim3((unsigned)((per + 255) / 256), (unsigned)B), 256, 0, c.stream>>>(s.utt, mel, m.n_mels, m.n_mels, m.eps, m.log10, mel_out);
    SSB_CUDA(cudaGetLastError());
    ++g_launches;
  }
  return 0;
}

}  // namespace

}  // namespace ssb

using namespace ssb;

extern "C" {

int ssb_melspec_create(ssb_melspec_t** out, int32_t sample_rate, int32_t fft_size, int32_t hop_size, int32_t win_length,
                       int32_t n_mels, float fmin, float fmax, float eps) {
  return ssb_melspec_create_ex(out, sample_rate, fft_size, hop_size, win_length, n_mels, fmin, fmax, eps, 0, 0, 1);
}

int ssb_melspec_create_ex(ssb_melspec_t** out, int32_t sample_rate, int32_t fft_size, int32_t hop_size, int32_t win_length,
                          int32_t n_mels, float fmin, float fmax, float eps, int32_t pad_reflect, int32_t power, int32_t take_log) {
  SSB_CHECK(out, "null argument");
  *out = nullptr;
  SSB_CHECK(sample_rate > 0 && fft_size > 0 && hop_size > 0 && win_length > 0 && win_length <= fft_size && n_mels > 0, "bad front-end geometry");
  SSB_CHECK(fft_size % 2 == 0 && hop_size % 16 == 0, "the implicit-GEMM STFT needs an even n_fft and hop_size a multiple of 16");
  // frame = `taps` whole rows of hop samples centred on sample t * hop: span = n_fft rounded up to a multiple of 2 hop, the
  // DFT weights of the `lead` samples in front of / behind the n_fft window are zero
  const int span = stft_span(fft_size, hop_size);
  // the frame reaches taps / 2 rows into the guard band on either side; with reflect centring both neighbours WRITE their
  // pads into the guard rows they share, so the two pads together must fit
  SSB_CHECK(span / hop_size / 2 <= (pad_reflect ? GUARD / 2 : GUARD), "n_fft / hop_size too large for the guard band");
  SSB_CHECK(n_mels % 4 == 0, "n_mels must be a multiple of 4");
  std::unique_ptr<ssb_melspec> m(new ssb_melspec);
  m->sample_rate = sample_rate; m->n_fft = fft_size; m->hop = hop_size; m->win = win_length; m->n_mels = n_mels;
  m->nbins = fft_size / 2 + 1;
  m->nbp = (m->nbins + 15) & ~15;
  m->taps = span / hop_size;
  m->eps = eps;
  m->reflect = pad_reflect ? 1 : 0; m->power = power ? 1 : 0; m->log10 = take_log ? 1 : 0;
  if (fmin < 0) fmin = 0.f;                       // librosa_wav2spec: fmin == -1 -> 0, fmax == -1 -> sr / 2
  if (fmax < 0) fmax = 0.5f * (float)sample_rate;
  const int N2 = 2 * m->nbp;
  m->dft.W = m->pool.upload(dft_basis(fft_size, hop_size, win_length, m->nbp, false));
  m->dft.bias = nullptr;
  m->dft.taps = m->taps; m->dft.Cin = hop_size; m->dft.N = N2; m->dft.Npad = N2; m->dft.dil = 1; m->dft.center = m->taps / 2;
  // mel basis (librosa.filters.mel, Slaney)
  std::vector<double> mel_f((size_t)n_mels + 2);
  const double m0 = hz_to_mel(fmin), m1 = hz_to_mel(fmax);
  for (int i = 0; i < n_mels + 2; ++i) mel_f[(size_t)i] = mel_to_hz(m0 + (m1 - m0) * i / (n_mels + 1));
  std::vector<float> Mb((size_t)m->nbp * n_mels, 0.f);  // [c = bin][n = mel]
  for (int i = 0; i < n_mels; ++i) {
    const double enorm = 2.0 / (mel_f[(size_t)i + 2] - mel_f[(size_t)i]);
    for (int k = 0; k < m->nbins; ++k) {
      const double f = (double)k * sample_rate / fft_size;  // np.linspace(0, sr / 2, 1 + n_fft // 2)
      const double lower = (f - mel_f[(size_t)i]) / (mel_f[(size_t)i + 1] - mel_f[(size_t)i]);
      const double upper = (mel_f[(size_t)i + 2] - f) / (mel_f[(size_t)i + 2] - mel_f[(size_t)i + 1]);
      const double v = std::max(0.0, std::min(lower, upper)) * enorm;
      Mb[(size_t)k * n_mels + i] = (float)v;
    }
  }
  m->mel.W = m->pool.upload(Mb);
  m->mel.bias = nullptr;
  m->mel.taps = 1; m->mel.Cin = m->nbp; m->mel.N = n_mels; m->mel.Npad = n_mels; m->mel.dil = 1; m->mel.center = 0;
  SSB_CHECK(m->dft.W && m->mel.W, "device allocation failed");
  *out = m.release();
  return 0;
}
void ssb_melspec_free(ssb_melspec_t* m) { delete m; }

int32_t ssb_melspec_num_frames(const ssb_melspec_t* m, int64_t n_samples) { return m && n_samples >= 0 ? frames_of(n_samples, m->hop) : 0; }

size_t ssb_melspec_workspace_bytes(const ssb_melspec_t* m, const int32_t* sample_offsets, int32_t B) {
  if (!m || !sample_offsets || B < 0) return 0;
  Ctx c;
  c.dry = true;
  Seq q;
  if (build_seq(sample_offsets, B, m->hop, &q) != 0) return 0;
  if (run_melspec(c, *m, q, nullptr, sample_offsets, B, nullptr) != 0) return 0;
  return c.high + 4096;
}

int ssb_melspec_forward(const ssb_melspec_t* m, const float* wav, const int32_t* sample_offsets, int32_t B, float* mel_out,
                        void* workspace, size_t workspace_bytes, void* stream) {
  SSB_CHECK(m && sample_offsets && workspace && B >= 0, "bad argument");
  // an empty tensor may have no storage: no samples in the batch need no waveform pointer, no utterance no output
  SSB_CHECK(wav || sample_offsets[B] == sample_offsets[0], "null waveform");
  SSB_CHECK(mel_out || B == 0, "null output");
  Ctx c;
  c.base = (char*)workspace; c.cap = workspace_bytes; c.stream = (cudaStream_t)stream;
  Seq q;
  RUN(build_seq(sample_offsets, B, m->hop, &q));
  return run_melspec(c, *m, q, wav, sample_offsets, B, mel_out);
}

}  // extern "C"
