"""ORACLE - test infrastructure only.  NOT part of the product path.

float64 restatement of the reference's vocoder output denoiser, denoise(wav, v) of tasks/tts/vocoder_infer/hifigan_nsf.py:14-22
(also vocoders/vocoder_utils.py:7-15), which HifiGAN.spec2wav applies when hparams['vocoder_denoise_c'] > 0.  Its arithmetic
lives in librosa 0.8.0 (requirements.txt:2), which is neither vendored in the reference nor installed here: `stft`, `istft`
and `window_sumsquare` below restate librosa 0.8.0's published algorithms.  PARITY UNPINNED against librosa itself; the
independent check is tests/test_wav_denoise_cpu.py, which compares `denoise` with torch.stft / torch.istft.
"""
import numpy as np

from oracle.frontend_oracle import hann_periodic, pad_center


def stft(y, n_fft, hop_length, win_length):
    """librosa.stft(y, n_fft, hop_length, win_length, window='hann', center=True, pad_mode='constant') in float64:
    complex [1 + n_fft/2, 1 + len(y) // hop_length]."""
    y = np.asarray(y, dtype=np.float64)
    w = pad_center(hann_periodic(win_length), n_fft).reshape(-1, 1)
    yp = np.pad(y, n_fft // 2, mode="constant")
    n_frames = 1 + (len(yp) - n_fft) // hop_length
    idx = np.arange(n_fft)[:, None] + hop_length * np.arange(n_frames)[None, :]
    return np.fft.rfft(w * yp[idx], axis=0)


def window_sumsquare(n_frames, hop_length, win_length, n_fft):
    """librosa.filters.window_sumsquare(window='hann', norm=None): sum over the frames of the squared (padded) window,
    length n_fft + hop_length (n_frames - 1)."""
    x = np.zeros(n_fft + hop_length * (n_frames - 1))
    win_sq = pad_center(hann_periodic(win_length) ** 2, n_fft)
    for i in range(n_frames):
        s = i * hop_length
        x[s:min(len(x), s + n_fft)] += win_sq[:max(0, min(n_fft, len(x) - s))]
    return x


def istft(S, hop_length, win_length):
    """librosa.istft(S, hop_length, win_length, window='hann', center=True, length=None) in float64: n_fft = 2 (bins - 1);
    irfft of every frame times the window, overlap-add, division by the window sum-square where it exceeds tiny(float32)
    (librosa passes the float32 output array to util.tiny), n_fft / 2 trimmed from each end."""
    n_fft = 2 * (S.shape[0] - 1)
    w = pad_center(hann_periodic(win_length), n_fft)[:, None]
    n_frames = S.shape[1]
    frames = w * np.fft.irfft(S, n=n_fft, axis=0)
    y = np.zeros(n_fft + hop_length * (n_frames - 1))
    for t in range(n_frames):
        y[t * hop_length:t * hop_length + n_fft] += frames[:, t]
    wss = window_sumsquare(n_frames, hop_length, win_length, n_fft)
    nz = wss > np.finfo(np.float32).tiny
    y[nz] /= wss[nz]
    return y[n_fft // 2:-(n_fft // 2)]


def subtract(S, v):
    """max(|S| - v, 0) * exp(i angle(S)) (hifigan_nsf.py:17-21); np.angle(0) = 0."""
    return np.clip(np.abs(S) - v, 0, None) * np.exp(1j * np.angle(S))


def denoise(wav, v, n_fft=1024, hop=256, win=1024):
    """denoise(wav, v) of hifigan_nsf.py:14-22 with hparams fft_size / hop_size / win_size = n_fft / hop / win."""
    return istft(subtract(stft(wav, n_fft, hop, win), v), hop, win)
