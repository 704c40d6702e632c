"""CPU checks of the vocoder output denoiser (hparams['vocoder_denoise_c'], tasks/tts/vocoder_infer/hifigan_nsf.py:14-22):
the float64 oracle against an independent STFT / ISTFT (torch), the C ABI's argument checks, and that the default
configuration leaves the denoiser out."""
import ctypes

import numpy as np
import pytest
import torch

from tests import wav_denoise_oracle as WO

N_FFT, HOP, WIN = 1024, 256, 1024


def _wave(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 48000.0
    x = 0.3 * np.sin(2 * np.pi * 440.0 * t) + 0.2 * np.sin(2 * np.pi * 1234.5 * t + 1.0) + 0.01 * rng.standard_normal(n)
    return np.clip(x, -1.0, 1.0).astype(np.float32)


def _torch_denoise(wav, v, n_fft=N_FFT, hop=HOP, win=WIN):
    """The same computation on torch.stft / torch.istft in float64 (window = periodic Hann of `win`, which torch pads to
    n_fft centred like librosa), the subtraction between the two calls."""
    w = torch.hann_window(win, periodic=True, dtype=torch.float64)
    x = torch.from_numpy(np.asarray(wav, np.float64))
    S = torch.stft(x, n_fft, hop, win, window=w, center=True, pad_mode="constant", return_complex=True)
    mag = S.abs()
    S = torch.clamp(mag - v, min=0) * torch.exp(1j * torch.angle(S))
    return torch.istft(S, n_fft, hop, win, window=w, center=True, length=None).numpy()


@pytest.mark.parametrize("frames", [1, 2, 3, 4, 5, 300])
@pytest.mark.parametrize("v", [0.0, 0.01, 0.1, 1.0])
def test_oracle_matches_torch_stft_istft(frames, v):
    wav = _wave(frames * HOP, seed=frames)
    ref = _torch_denoise(wav, v)
    got = WO.denoise(wav, v, N_FFT, HOP, WIN)
    assert got.shape == (frames * HOP,) == ref.shape
    assert np.abs(got - ref).max() < 1e-12


@pytest.mark.parametrize("frames", [1, 2, 5, 300])
def test_oracle_round_trip_at_zero_strength(frames):
    wav = _wave(frames * HOP, seed=7 + frames)
    assert np.abs(WO.denoise(wav, 0.0, N_FFT, HOP, WIN) - wav).max() < 1e-12


def test_oracle_short_window():
    """win_size < fft_size: the window is zero-padded to n_fft (librosa.util.pad_center), as torch does it."""
    wav = _wave(6 * 128, seed=3)
    assert np.abs(WO.denoise(wav, 0.05, 512, 128, 400) - _torch_denoise(wav, 0.05, 512, 128, 400)).max() < 1e-12


def test_denoiser_argument_checks_need_no_gpu():
    """Geometry and argument validation happen before any CUDA call: same error behaviour on any host."""
    from stylesinger_b200 import _lib
    lib, C = _lib.lib, ctypes
    h = C.c_void_p()
    # odd n_fft, hop not a multiple of 16, win > n_fft, n_fft too long for the guard band, non-positive sizes
    for args in ((1023, 256, 1023), (1024, 250, 1024), (1024, 256, 1025), (40 * 256, 256, 1024), (0, 256, 0),
                 (1024, 0, 1024), (1024, 256, 0)):
        assert lib.ssb_wav_denoise_create(C.byref(h), *args) != 0 and not h.value, args
    assert lib.ssb_wav_denoise_create(None, 1024, 256, 1024) != 0
    offs = np.array([0, 256, 512], np.int32)
    assert lib.ssb_wav_denoise_workspace_bytes(None, offs.ctypes.data, 2) == 0
    assert lib.ssb_wav_denoise_forward(None, None, offs.ctypes.data, 2, C.c_float(0.1), None, None, 0, None) != 0
    assert lib.ssb_wav_denoise_set_tensor_cores(None, 1) != 0
    lib.ssb_wav_denoise_free(None)


def test_default_configuration_has_no_denoiser():
    from stylesinger_b200 import modules
    from stylesinger_b200.hparams import resolve
    assert resolve()["vocoder_denoise_c"] == 0.0

    class _Engine:  # records what HifiGAN.spec2wav asks the vocoder for
        device = torch.device("cpu")

        def generate(self, mel, f0, offs, seed=0, denoise_c=None):
            self.denoise_c = denoise_c
            return torch.zeros(int(offs[-1]) * 256)

    e = _Engine()
    modules.HifiGAN(engine=e).spec2wav(np.zeros((3, 80), np.float32))
    assert e.denoise_c == 0.0
    modules.HifiGAN(engine=e, denoise_c=0.1).spec2wav(np.zeros((3, 80), np.float32))
    assert e.denoise_c == 0.1
