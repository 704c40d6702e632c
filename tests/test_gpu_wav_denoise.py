"""The vocoder output denoiser (hparams['vocoder_denoise_c'], tasks/tts/vocoder_infer/hifigan_nsf.py:14-22,73-74) on the GPU
against the float64 oracle (tests/wav_denoise_oracle.py): both GEMM paths on a ragged batch with 1..5-frame utterances, the
batch64 lengths on the automatic path, B = 1 semantics, in-place calls, the workspace contract, and the inference driver.

Bars (L-inf, waveform in [-1, 1]): 1e-5 for the fp32 FFMA GEMMs, 5e-5 for the 3-pass fp16 hi/lo tensor-core GEMMs (about
22 mantissa bits per product; the spectrum of a loud sinusoid reaches ~150, so its fp16 lo plane carries ~3e-5 absolute).
"""
import ctypes as C

import numpy as np
import pytest
import torch

from stylesinger_b200 import _lib
from tests import wav_denoise_oracle as WO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HOP = 256
BAR_FFMA = 1e-5
BAR_TC = 5e-5
RAGGED = [300, 1, 250, 2, 3, 4, 5, 200]  # frames; a 1-frame utterance between two long ones; 12 row tiles


def _waves(frames, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i, F in enumerate(frames):
        n = F * HOP
        t = np.arange(n) / 48000.0
        f1, f2 = 110.0 * (1 + i % 7), 1234.5 + 37.0 * i
        x = (0.3 * np.sin(2 * np.pi * f1 * t) + 0.2 * np.sin(2 * np.pi * f2 * t + i) + 1e-3 * rng.standard_normal(n)
             + 0.05 * rng.standard_normal(n) * (rng.random(n) < 0.01))
        out.append(np.clip(x, -1.0, 1.0).astype(np.float32))
    return out


def _offs(wavs):
    return np.concatenate([[0], np.cumsum([len(w) for w in wavs])]).astype(np.int32)


def _generic_tc_launches():
    return sum(n for k, n in _lib.variant_launches().items() if "GENERIC" in k)


def _denoiser():
    from stylesinger_b200.engine import WavDenoiser
    return WavDenoiser(None, DEV)


def _max_err(out, wavs, offs, v):
    o = out.cpu().numpy().astype(np.float64)
    return max(float(np.abs(o[offs[i]:offs[i + 1]] - WO.denoise(w, v)).max()) for i, w in enumerate(wavs))


def test_ragged_batch_both_paths_match_the_oracle():
    d = _denoiser()
    wavs = _waves(RAGGED, seed=1)
    offs = _offs(wavs)
    x = torch.from_numpy(np.concatenate(wavs)).to(DEV)
    for v in (0.0, 0.01, 0.1):
        S = np.concatenate([np.abs(WO.stft(w, 1024, HOP, 1024)).ravel() for w in wavs])
        clipped = float((S <= v).mean())
        print(f"v={v}: clipped bins {clipped:.3f}, unclipped {1 - clipped:.3f}")
        if v > 0:
            assert 0.0 < clipped < 1.0
        errs = {}
        for tc in (False, True):
            assert d.set_tensor_cores(2 if tc else 0) == (2 if tc else 0)  # forced
            n0 = _generic_tc_launches()
            out = d(x, offs, v)
            torch.cuda.synchronize()
            n1 = _generic_tc_launches()
            if tc:
                assert n1 - n0 == 2, "tensor-core arm: both DFT GEMMs on GENERIC tensor-core variants"
            else:
                assert n1 == n0, "FFMA arm launched a tensor-core variant"
            errs["tc" if tc else "ffma"] = _max_err(out, wavs, offs, v)
        print(f"v={v}: L-inf error FFMA {errs['ffma']:.3e} (bar {BAR_FFMA}), tensor cores {errs['tc']:.3e} (bar {BAR_TC})")
        assert errs["ffma"] < BAR_FFMA and errs["tc"] < BAR_TC


def test_bench_sized_batch_takes_tensor_cores_and_matches_the_oracle():
    from bench import make_workload
    utts, _ = make_workload("batch64", 0, 1)
    frames = [len(u["mel2ph"]) for u in utts]
    wavs = _waves(frames, seed=2)
    offs = _offs(wavs)
    print(f"batch64: {len(frames)} utterances, {int(offs[-1])} samples")
    d = _denoiser()
    x = torch.from_numpy(np.concatenate(wavs)).to(DEV)
    n0 = _generic_tc_launches()
    out = d(x, offs, 0.1)
    torch.cuda.synchronize()
    assert _generic_tc_launches() - n0 == 2
    err = _max_err(out, wavs, offs, 0.1)
    print(f"batch64, v=0.1: L-inf error {err:.3e} (bar {BAR_TC})")
    assert err < BAR_TC


def test_every_utterance_matches_its_own_call():
    """Mode 0: batch and solo calls on the FFMA kernel, bit-identical.  Mode 1 (automatic): the 12-row-tile batch takes
    tensor cores, every solo call (at most 3 row tiles) FFMA."""
    d = _denoiser()
    wavs = _waves(RAGGED, seed=3)
    offs = _offs(wavs)
    x = torch.from_numpy(np.concatenate(wavs)).to(DEV)
    for mode in (0, 1):
        assert d.set_tensor_cores(mode) == mode
        n0 = _generic_tc_launches()
        batch = d(x, offs, 0.05).cpu().numpy()
        assert _generic_tc_launches() - n0 == (2 if mode else 0)
        worst = 0.0
        for i, w in enumerate(wavs):
            n0 = _generic_tc_launches()
            solo = d(torch.from_numpy(w).to(DEV), [0, len(w)], 0.05).cpu().numpy()
            assert _generic_tc_launches() == n0, "a solo call below 8 row tiles took tensor cores"
            part = batch[offs[i]:offs[i + 1]]
            if mode == 0:
                assert np.array_equal(part, solo), i
            worst = max(worst, float(np.abs(part.astype(np.float64) - solo).max()))
        print(f"mode {mode}: batch vs solo L-inf {worst:.3e}")
        assert worst < (BAR_FFMA if mode == 0 else BAR_TC)


def test_in_place_and_workspace_contract():
    d = _denoiser()
    wavs = _waves(RAGGED, seed=4)
    offs = _offs(wavs)
    x = torch.from_numpy(np.concatenate(wavs)).to(DEV)
    ref = d(x, offs, 0.1)
    y = x.clone()
    assert d(y, offs, 0.1, out=y) is y
    assert torch.equal(y, ref)
    lib = _lib.lib
    n = d.workspace_bytes(offs)
    assert n > 0
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    out = torch.empty_like(x)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    call = lambda v, nbytes, o=offs: lib.ssb_wav_denoise_forward(d._h, C.c_void_p(x.data_ptr()), o.ctypes.data, len(o) - 1,
                                                                 C.c_float(v), C.c_void_p(out.data_ptr()),
                                                                 C.c_void_p(ws.data_ptr()), nbytes, stream)
    assert call(0.1, n - 1) != 0 and b"workspace too small" in lib.ssb_last_error()
    assert call(-0.1, n) != 0 and call(float("nan"), n) != 0 and call(float("inf"), n) != 0
    assert call(0.1, n) == 0
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    bad = np.array([0, 256, 256 + 300], np.int32)  # a length that is not a multiple of hop_size
    assert d.workspace_bytes(bad) == 0 and call(0.1, n, bad) != 0
    assert d.workspace_bytes(np.array([0, 0], np.int32)) == 0  # an empty utterance


def _infer_engines(c):
    from stylesinger_b200 import synth
    from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG
    from stylesinger_b200.infer import StyleSingerInfer
    from tests.common import acoustic_sd, hp_for, vocoder_sd
    hp = hp_for(4)
    assert hp["vocoder_denoise_c"] == 0.0
    e0 = StyleSingerInfer(hp, DEV, acoustic_sd(), vocoder_sd(), DEFAULT_VOCODER_CONFIG)
    e1 = StyleSingerInfer(dict(hp, vocoder_denoise_c=c), DEV, acoustic_sd(), vocoder_sd(), DEFAULT_VOCODER_CONFIG)
    return e0, e1, synth


def test_inference_driver_applies_the_denoiser_only_when_asked():
    from stylesinger_b200.engine import pack_batch
    from stylesinger_b200.modules import HifiGAN
    from tests.common import batch_noise, engine_noise_from_stream
    e0, e1, synth = _infer_engines(0.1)
    specs = [(90, 8, 40, 31), (17, 4, 20, 32), (61, 7, 30, 33)]  # frames, phones, ref frames, utt_idx
    utts = [synth.make_utterance(f / 187.5, utt_idx=i, ref_frames=r, frames=f, phones=p) for f, p, r, i in specs]
    noise = batch_noise([engine_noise_from_stream(900 + k, 4, 4, u["mel2ph"].shape[0], DEV)[0] for k, u in enumerate(utts)])
    F = sum(int(u["mel2ph"].shape[0]) for u in utts)
    g = torch.Generator().manual_seed(5)
    voc = {"rand_ini": torch.rand(len(utts), 9, generator=g).to(DEV), "src_noise": torch.randn(F * HOP, 9, generator=g).to(DEV)}
    mel0, f00, wav0, fo0 = e0.run_device(pack_batch(utts).to(DEV), noise=noise, voc_noise=voc)
    # the default configuration creates no denoiser (so none of its kernels can run), and its waveform is the generator's
    assert e0.vocoder._denoiser is None
    melc = mel0.clamp(e0.hparams["mel_vmin"], e0.hparams["mel_vmax"]).contiguous()  # ssb_mel_postprocess
    l2 = _lib.lib.ssb_launch_count()
    raw = e0.vocoder.generate(melc, f00, fo0, rand_ini=voc["rand_ini"], src_noise=voc["src_noise"])
    torch.cuda.synchronize()
    l3 = _lib.lib.ssb_launch_count()
    assert torch.equal(wav0, raw)
    mel1, _, wav1, fo1 = e1.run_device(pack_batch(utts).to(DEV), noise=noise, voc_noise=voc)
    torch.cuda.synchronize()
    assert torch.equal(mel0, mel1) and np.array_equal(fo0, fo1)
    assert e1.vocoder._denoiser is not None
    w0, w1 = wav0.cpu().numpy(), wav1.cpu().numpy()
    worst = 0.0
    for b in range(len(utts)):
        s = slice(int(fo0[b]) * HOP, int(fo0[b + 1]) * HOP)
        worst = max(worst, float(np.abs(w1[s] - WO.denoise(w0[s], 0.1)).max()))
    print(f"StyleSingerInfer, vocoder_denoise_c=0.1: L-inf vs oracle.denoise of the undenoised run {worst:.3e}")
    assert worst < BAR_FFMA
    # a per-call strength of 0 on the denoising engine launches exactly what the plain vocoder launches
    l4 = _lib.lib.ssb_launch_count()
    e1.vocoder.generate(melc, f00, fo0, rand_ini=voc["rand_ini"], src_noise=voc["src_noise"], denoise_c=0.0)
    torch.cuda.synchronize()
    assert _lib.lib.ssb_launch_count() - l4 == l3 - l2
    # modules.HifiGAN: the key taken like use_nsf
    m, f = melc[:int(fo0[1])].cpu().numpy(), f00[:int(fo0[1])].cpu().numpy()
    plain = HifiGAN(engine=e0.vocoder).spec2wav(m, f0=f, seed=3)
    den = HifiGAN(engine=e0.vocoder, denoise_c=0.1).spec2wav(m, f0=f, seed=3)
    err = float(np.abs(den - WO.denoise(plain, 0.1)).max())
    print(f"HifiGAN.spec2wav, denoise_c=0.1: L-inf vs oracle {err:.3e}")
    assert err < BAR_FFMA
