"""The reference-audio front-end against float64: the mel spectrogram (ssb_melspec_*, csrc/frontend.cu) in both of its
configurations, the cluster LSTM (ssb_lstm_encoder_*, csrc/lstm.cu) at batch scale, and the two encoders built on them
(stylesinger_b200.voice_encoder.VoiceEncoder, stylesinger_b200.emotion).

The mel spectrogram is checked element by element against the bound of tests/frontend_ref.py, which grows with the frame's
windowed L1 norm rather than with the band's own value, so it holds for any signal: silence gaps, onsets, clipping, DC,
impulses, bands far below the loudest one.  Configurations: librosa_wav2spec at 48 kHz (zero centring, |X|, log10; and the
same geometry without the log, so that a wrong value cannot hide under the eps floor) and the encoders' 16 kHz features
(reflect centring, n_fft 400 over hop 160, |X|^2, no log).

ALPHA / BETA of each configuration are at no more than 4x the smallest values that cover every element measured on an
H100 80GB HBM3 (SXM, 700 W power limit), written beside them; each test prints err / bound.  The LSTM bars are those of
tests/test_gpu_emotion.py, with the errors measured at batch scale beside them.
"""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import frontend_oracle as FO
from stylesinger_b200 import synth
from tests import frontend_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (alpha, beta) per configuration, measured beside them (tests/frontend_ref.calibrate over every test of the file); the
# two 48 kHz configurations run the same kernels, the log one is bounded through the linear one's constants
BOUND = {
    "wav2spec": (5e-7, 2.3e-5),
    "wav2spec_lin": (5e-7, 2.3e-5),   # alpha 1.47e-7, beta 5.76e-6
    "emotion": (3e-7, 9.9e-6),        # alpha 7.73e-8, beta 2.48e-6
}
CONFIGS = tuple(BOUND)
LSTM_BARS = {"hidden": 1e-6,   # 2.1e-7 at batch scale, inputs up to 1.3e2
             "embeds": 2e-6,   # 2.4e-7
             "utt": 1e-6}      # 6.2e-8
ENCODER_BAR = 2e-6   # encoder outputs of the CUDA mel + LSTM against the float64 composition: 2.2e-7


def _edges(cfg):
    c = R.CONFIGS[cfg]
    hop, n_fft = c["hop"], c["n_fft"]
    return [1, 2, hop - 1, hop, hop + 1, n_fft // 2, n_fft // 2 + 1, n_fft - 1, n_fft, n_fft + 1, 17 * hop - 1, 17 * hop]


def _launches():
    from stylesinger_b200 import _lib
    return int(_lib.lib.ssb_launch_count())


def _check_all(fe_out, wavs, cfg, tag):
    """Every utterance inside the bound; returns the worst err / bound and the calibration of the linear configurations."""
    alpha, beta = BOUND[cfg]
    worst, cal = 0.0, (0.0, 0.0)
    for i, (m, y) in enumerate(zip(fe_out, wavs)):
        ratio, (A, B, err) = R.check(m.cpu().numpy(), y, cfg, alpha, beta)
        if err is not None and err.size:
            a, b = R.calibrate(A, B, err)
            cal = (max(cal[0], a), max(cal[1], b))
        assert ratio <= 1.0, f"{cfg} {tag}: utterance {i} (n={len(y)}) err / bound {ratio:.3f}"
        worst = max(worst, ratio)
    return worst, cal


def _report(cfg, tag, worst, cal):
    extra = f", measured alpha {cal[0]:.2e} beta {cal[1]:.2e}" if not R.CONFIGS[cfg]["log"] else ""
    print(f"melspec {cfg} {tag}: max err / bound {worst:.3f}{extra}")


@pytest.mark.parametrize("cfg", CONFIGS)
def test_melspec_signals_against_float64(cfg):
    c = R.CONFIGS[cfg]
    fe = R.melspec(cfg, DEV)
    n = int(1.5 * c["sr"]) + 77
    wavs = [R.signal(k, n, c["sr"], c["hop"], seed=i) for i, k in enumerate(R.KINDS)]
    out = fe(wavs)
    worst, cal = 0.0, (0.0, 0.0)
    for k, y, m in zip(R.KINDS, wavs, out):
        w, cl = _check_all([m], [y], cfg, k)
        worst, cal = max(worst, w), (max(cal[0], cl[0]), max(cal[1], cl[1]))
    _report(cfg, "signals", worst, cal)
    z = out[R.KINDS.index("zeros")]
    floor = float(np.log10(c["eps"])) if c["log"] else 0.0   # exactly -6.0 / 0.0
    assert torch.equal(z, torch.full_like(z, floor)), "silence must be exactly the floor"


@pytest.mark.parametrize("cfg", CONFIGS)
def test_melspec_length_edges_in_one_ragged_call(cfg):
    """Every edge length of the configuration in one ragged call, interleaved with 6 s clips: each against float64 and
    bit-identical to its own solo call (in reflect mode the pads of neighbours share guard rows).  Zero centring also takes
    an empty utterance (one frame at the floor, as np.pad of an empty array gives)."""
    c = R.CONFIGS[cfg]
    fe = R.melspec(cfg, DEV)
    kinds = ("noise", "sweep", "gaps", "square")
    edges = _edges(cfg) + ([] if c["reflect"] else [0])
    wavs = []
    for i, n in enumerate(edges):
        if i % 2 == 0:
            wavs.append(R.signal(kinds[i // 2 % 4], 6 * c["sr"], c["sr"], c["hop"], seed=100 + i))
        wavs.append(R.signal(kinds[i % 4], n, c["sr"], c["hop"], seed=i))
    out = fe(wavs)
    assert [tuple(m.shape) for m in out] == [(1 + len(y) // c["hop"], c["n_mels"]) for y in wavs]
    worst, cal = _check_all(out, wavs, cfg, "edges")
    _report(cfg, "length edges", worst, cal)
    for i, y in enumerate(wavs):
        assert torch.equal(fe(y), out[i]), f"utterance {i} (n={len(y)}) differs from its solo call"
    if not c["reflect"]:
        e = out[[len(y) for y in wavs].index(0)]
        assert e.shape[0] == 1 and torch.equal(e, torch.full_like(e, float(np.log10(c["eps"])) if c["log"] else 0.0))


def test_reflect_centring_refuses_only_an_empty_utterance():
    from stylesinger_b200 import _lib
    fe = R.melspec("emotion", DEV)
    y = R.signal("noise", 3000, 16000, 160)
    fe([y])
    torch.cuda.synchronize()
    n0 = _launches()
    for batch in ([np.zeros(0, np.float32)], [y, np.zeros(0, np.float32), y]):
        with pytest.raises(_lib.SsbError, match="at least one sample"):
            fe(batch)
    assert _launches() == n0, "a refused call launched kernels"
    # every reflect length up to n_fft / 2 (numpy reflects as often as the pad needs) matches float64
    wavs = [R.signal("noise", n, 16000, 160, seed=n) for n in range(1, 201)]
    worst, cal = _check_all(fe(wavs), wavs, "emotion", "short")
    _report("emotion", "n = 1 .. 200", worst, cal)


def test_melspec_empty_batch():
    for cfg in ("wav2spec", "emotion"):
        assert R.melspec(cfg, DEV)([]) == []


@functools.lru_cache(maxsize=None)
def _bench_clips(sr):
    """The bench's batch64 durations (2 - 15 s) at sample rate sr: speech with pauses, tones, noise, float16 input."""
    kinds = ("gaps", "sweep", "gaps", "noise", "gaps", "f16")
    return tuple(R.signal(kinds[i % len(kinds)], int(round(s * sr)), sr, 160, seed=1000 + i)
                 for i, s in enumerate(synth.batch_seconds(64, seed=1234)))


@pytest.mark.parametrize("cfg", CONFIGS)
def test_melspec_bench_batch_against_float64(cfg):
    c = R.CONFIGS[cfg]
    fe = R.melspec(cfg, DEV)
    wavs = list(_bench_clips(c["sr"]))
    dev_wavs = [torch.as_tensor(np.asarray(y, np.float32), device=DEV) for y in wavs]
    out = fe(dev_wavs)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(5):
        fe(dev_wavs)
    ev[1].record()
    torch.cuda.synchronize()
    frames = sum(m.shape[0] for m in out)
    print(f"melspec {cfg} batch64: {sum(len(y) for y in wavs)} samples, {frames} frames, "
          f"{ev[0].elapsed_time(ev[1]) / 5:.3f} ms per call ({torch.cuda.get_device_name()})")
    worst, cal = _check_all(out, wavs, cfg, "batch64")
    _report(cfg, "batch64", worst, cal)


# ---- the LSTM at batch scale --------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _partials():
    """The emotion-mel partials of the batch64 clips at 16 kHz, cut as emotion.embed_utterance cuts them (zero-padded to the
    end of the last partial), from the float64 power mel; with the per-clip partial offsets.  The clips are scaled to a
    full-scale voice (peaks near 1), whose power mel reaches 1e2 and saturates the gates."""
    from stylesinger_b200 import emotion
    frames, offs = [], [0]
    for y in _bench_clips(16000):
        y = 3.0 * np.asarray(y, np.float32)
        wav_sl, mel_sl = emotion.compute_partial_slices(len(y))
        yp = np.pad(y, (0, max(0, wav_sl[-1].stop - len(y))))
        mel = R.reference(yp, "emotion", 0.0, 0.0)[0].astype(np.float32)
        frames += [mel[s] for s in mel_sl]
        offs.append(len(frames))
    return np.stack(frames), np.array(offs, np.int32)


def _lstm_weights():
    sd = FO.emotion_encoder_weights(5)
    for k in list(sd):  # larger recurrent weights: states leave the linear regime of the gates
        if "weight_hh" in k:
            sd[k] = (sd[k] * 3.0).astype(np.float32)
    return sd


def test_lstm_encoder_bench_batch_against_float64():
    from stylesinger_b200.engine import LstmEncoder
    x, offs = _partials()
    P = x.shape[0]
    assert x.shape[1:] == (160, 40) and P > 8 * 32 and P % 8 != 0, "want tens of clusters and a ragged last one"
    sd = _lstm_weights()
    enc = LstmEncoder(sd, DEV)
    out = enc(x, utt_offsets=offs, want_embeds=True)
    torch.cuda.synchronize()
    ref = R.lstm_hidden64(x, sd)
    dh = np.abs(out["hidden"].cpu().numpy() - ref).max()
    de = np.abs(out["embeds"].cpu().numpy() - R.embeds64(ref, sd)).max()
    du = max(np.abs(out["utt_embed"][u].cpu().numpy() - R.utt_embed64(ref[offs[u]:offs[u + 1]])).max() for u in range(len(offs) - 1))
    print(f"lstm batch64: {P} partials x 160 frames ({(P + 7) // 8} clusters), input max {x.max():.1f}: "
          f"hidden {dh:.3e}, embeds {de:.3e}, utterance {du:.3e}")
    assert dh < LSTM_BARS["hidden"] and de < LSTM_BARS["embeds"] and du < LSTM_BARS["utt"]
    # a partial's result does not depend on the batch: the first, the last, and one of the ragged last cluster
    for p in (0, P - 1, P - 2):
        solo = enc(x[p:p + 1], want_embeds=True)
        assert torch.equal(solo["hidden"][0], out["hidden"][p]) and torch.equal(solo["embeds"][0], out["embeds"][p]), p
    # the utterance embedding is the normalised MEAN: a group of two copies of a partial has exactly the bits of the
    # partial alone (h + h and its half are exact), whatever the rounding of the normalisation
    sel = [0, P // 2, P - 1]
    xs = np.stack([x[p] for p in sel for _ in range(3)])
    uo = np.array([0] + [v for j in range(len(sel)) for v in (3 * j + 1, 3 * j + 3)], np.int32)
    o2 = enc(xs, utt_offsets=uo)
    for j in range(len(sel)):
        assert torch.equal(o2["hidden"][3 * j], o2["hidden"][3 * j + 1]) and torch.equal(o2["hidden"][3 * j], o2["hidden"][3 * j + 2])
        assert torch.equal(o2["utt_embed"][2 * j], o2["utt_embed"][2 * j + 1]), sel[j]
        assert np.abs(o2["utt_embed"][2 * j].cpu().numpy() - R.utt_embed64(ref[sel[j]:sel[j] + 1])).max() < LSTM_BARS["utt"]


def test_lstm_encoder_refuses_too_many_rows_before_any_launch():
    from stylesinger_b200 import _lib
    from stylesinger_b200.engine import LstmEncoder
    enc = LstmEncoder(FO.emotion_encoder_weights(1), DEV)
    lib = _lib.lib
    torch.cuda.synchronize()
    n0 = _launches()
    assert lib.ssb_lstm_encoder_workspace_bytes(enc._h, 26214, 160, 1) > 0        # 4 194 240 rows: the limit
    assert lib.ssb_lstm_encoder_workspace_bytes(enc._h, 26215, 160, 1) == 0       # one partial more
    assert "too many frames" in lib.ssb_last_error().decode()
    assert lib.ssb_lstm_encoder_workspace_bytes(enc._h, 1, 4194241, 0) == 0
    assert _launches() == n0


# ---- the encoders ---------------------------------------------------------------------------------------------------------
def test_voice_encoder_against_the_float64_composition():
    """VoiceEncoder.embed_utterance (resemblyzer's algorithm on this package's kernels; PARITY UNPINNED against resemblyzer
    itself, which is not installed) against the same composition of float64 pieces: resemblyzer_partial_slices, the power
    mel, the LSTM, relu(linear) normalised, the normalised mean."""
    from stylesinger_b200.voice_encoder import VoiceEncoder
    sd = FO.emotion_encoder_weights(9)
    ve = VoiceEncoder(sd, DEV)
    cases = [R.signal("gaps", n, 16000, 160, seed=n) for n in (1, 25599, 37920, 160000)] + [R.signal("f16", 48000, 48000, 256, seed=3)]
    for y in cases:
        emb, partials, _ = ve.embed_utterance(y, return_partials=True)
        y32 = np.asarray(y, np.float32)
        wav_sl, mel_sl = FO.resemblyzer_partial_slices(len(y32))
        mel = R.reference(np.pad(y32, (0, max(0, wav_sl[-1][1] - len(y32)))), "emotion", 0.0, 0.0)[0]
        pe = R.embeds64(R.lstm_hidden64(np.stack([mel[a:b] for a, b in mel_sl]), sd), sd)
        raw = pe.mean(axis=0)
        dp, du = np.abs(partials - pe).max(), np.abs(emb - raw / np.linalg.norm(raw)).max()
        print(f"VoiceEncoder n={len(y)} ({y.dtype}): {len(mel_sl)} partials, partial embeds {dp:.3e}, utterance {du:.3e}")
        assert emb.shape == (256,) and dp < ENCODER_BAR and du < ENCODER_BAR


def test_emotion_embed_utterance_whole_short_clip():
    """embed_utterance(using_partials=False) runs the whole spectrogram as one sequence: a 150-sample clip is one reflect-
    padded frame, shorter than the pad on either side."""
    from stylesinger_b200 import emotion
    sd = FO.emotion_encoder_weights(4)
    emotion.load_model(sd, DEV)
    y = R.signal("noise", 150, 16000, 160, seed=150)
    whole = emotion.embed_utterance(y, using_partials=False)
    mel = R.reference(y, "emotion", 0.0, 0.0)[0]
    assert mel.shape == (1, 40)
    d = np.abs(whole - R.lstm_hidden64(mel[None], sd)[0]).max()
    print(f"emotion embed_utterance(using_partials=False), n=150: {d:.3e}")
    assert d < ENCODER_BAR


# ---- workspace contract ---------------------------------------------------------------------------------------------------
CANARY = 4096


def _short_workspace(nbytes):
    """A buffer of nbytes - 4097 usable bytes (the reported size includes 4096 bytes of slack) followed by a canary tail."""
    usable = nbytes - 4097
    buf = torch.zeros(usable + CANARY, dtype=torch.uint8, device=DEV)
    buf[usable:] = 0xA5
    return buf, usable


def test_workspace_one_byte_short_is_refused_without_writing_past_it():
    from stylesinger_b200 import _lib
    lib = _lib.lib
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    fe = R.melspec("emotion", DEV)
    wavs = [R.signal("noise", n, 16000, 160, seed=n) for n in (1, 16000, 3000)]
    offs = np.array([0, 1, 16001, 19001], np.int32)
    wav = torch.as_tensor(np.concatenate(wavs), device=DEV)
    out = torch.empty(sum(1 + len(y) // 160 for y in wavs), 40, device=DEV)
    n = lib.ssb_melspec_workspace_bytes(fe._h, offs.ctypes.data, 3)
    buf, usable = _short_workspace(n)
    torch.cuda.synchronize()
    n0 = _launches()
    rc = lib.ssb_melspec_forward(fe._h, wav.data_ptr(), offs.ctypes.data, 3, out.data_ptr(), buf.data_ptr(), usable, stream)
    torch.cuda.synchronize()
    assert rc != 0 and "workspace too small" in lib.ssb_last_error().decode()
    assert _launches() == n0 and bool((buf[usable:] == 0xA5).all())

    from stylesinger_b200.engine import LstmEncoder
    enc = LstmEncoder(FO.emotion_encoder_weights(1), DEV)
    x = torch.rand(11, 160, 40, device=DEV)
    uo = np.array([0, 4, 11], np.int32)
    hid = torch.empty(11, 256, device=DEV)
    emb = torch.empty(11, 256, device=DEV)
    utt = torch.empty(2, 256, device=DEV)
    n = lib.ssb_lstm_encoder_workspace_bytes(enc._h, 11, 160, 2)
    buf, usable = _short_workspace(n)
    torch.cuda.synchronize()
    n0 = _launches()
    rc = lib.ssb_lstm_encoder_forward(enc._h, x.data_ptr(), 11, 160, uo.ctypes.data, 2, hid.data_ptr(), emb.data_ptr(), utt.data_ptr(),
                                      buf.data_ptr(), usable, stream)
    torch.cuda.synchronize()
    assert rc != 0 and "workspace too small" in lib.ssb_last_error().decode()
    assert _launches() == n0 and bool((buf[usable:] == 0xA5).all())
