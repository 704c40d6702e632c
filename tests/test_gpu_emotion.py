"""f3 (emotion-encoder half): the cluster LSTM kernel and the librosa-default mel mode of the CUDA front-end.

Bars: LSTM outputs against the UNMODIFIED reference's EmotionEncoder (tests/golden/ref_emotion_encoder.npz, tools/make_golden.py)
and against the float64 restatement in oracle/frontend_oracle.py: |d hidden| < 1e-6 (fp32 FFMA, 480 dependent steps; torch's
own fp32 CPU LSTM sits 2e-8 from the float64 oracle).  Power mel against the numpy restatement of
librosa: |d| < 2e-5 of the loudest band (one fp32 GEMM with K = 640 per frame, errors relative to the frame's energy).
"""
import os

import numpy as np
import pytest
import torch

from oracle import frontend_oracle as FO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_emotion_encoder.npz")


def test_lstm_encoder_matches_the_reference_golden():
    from stylesinger_b200.engine import LstmEncoder
    g = np.load(GOLD)
    sd = FO.emotion_encoder_weights(int(g["seed"]))
    enc = LstmEncoder(sd, DEV)
    out = enc(g["frames"], utt_offsets=[0, 5], want_embeds=True)
    torch.cuda.synchronize()
    dh = np.abs(out["hidden"].cpu().numpy() - g["hidden"]).max()
    de = np.abs(out["embeds"].cpu().numpy() - g["embeds"]).max()
    du = np.abs(out["utt_embed"][0].cpu().numpy() - g["utt_embed"]).max()
    print(f"lstm vs reference: hidden {dh:.3e}, embeds {de:.3e}, utterance {du:.3e}")
    assert dh < 1e-6 and de < 2e-6 and du < 1e-6
    # device time of a 10 s utterance's worth of partials (12 x 160 frames), CUDA events on the launching stream
    x = torch.rand(12, 160, 40, device=DEV)
    for _ in range(3):
        enc(x, utt_offsets=[0, 12])
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(10):
        enc(x, utt_offsets=[0, 12])
    ev[1].record()
    torch.cuda.synchronize()
    print(f"lstm encoder, 12 partials x 160 frames: {ev[0].elapsed_time(ev[1]) / 10:.3f} ms per call")


def test_lstm_encoder_ragged_groups_and_utterances_match_the_oracle():
    from stylesinger_b200.engine import LstmEncoder
    sd = FO.emotion_encoder_weights(5)
    rng = np.random.default_rng(11)
    for k in list(sd):  # larger recurrent weights: states leave the linear regime of the gates
        if "weight_hh" in k:
            sd[k] = (sd[k] * 3.0).astype(np.float32)
    enc = LstmEncoder(sd, DEV)
    for P, T, offs in ((13, 37, [0, 4, 5, 13]), (1, 160, [0, 1]), (8, 3, [0, 8]), (17, 1, [0, 16, 17])):
        x = (rng.standard_normal((P, T, 40)) * 0.8).astype(np.float32)
        out = enc(x, utt_offsets=offs, want_embeds=True)
        ref = FO.lstm_hidden(x, sd)
        dh = np.abs(out["hidden"].cpu().numpy() - ref).max()
        de = np.abs(out["embeds"].cpu().numpy() - FO.emotion_embeds(ref, sd)).max()
        du = max(np.abs(out["utt_embed"][u].cpu().numpy() - FO.utterance_embed(ref[offs[u]:offs[u + 1]])).max() for u in range(len(offs) - 1))
        print(f"P={P} T={T}: hidden {dh:.3e}, embeds {de:.3e}, utterance {du:.3e}")
        assert dh < 1e-6 and de < 2e-6 and du < 1e-6
        # a partial's result does not depend on what shares its cluster
        solo = enc(x[P - 1:P])["hidden"]
        assert torch.equal(solo[0], out["hidden"][P - 1])


def test_lstm_encoder_error_behaviour():
    from stylesinger_b200 import _lib
    from stylesinger_b200.engine import LstmEncoder
    sd = FO.emotion_encoder_weights(1, hidden=128)
    with pytest.raises(_lib.SsbError, match="hidden_size 256"):
        LstmEncoder(sd, DEV)
    enc = LstmEncoder({k: v for k, v in FO.emotion_encoder_weights(1).items() if k.startswith("lstm.")}, DEV)
    x = np.zeros((2, 4, 40), np.float32)
    with pytest.raises(_lib.SsbError, match="linear head"):
        enc(x, want_embeds=True)
    with pytest.raises(_lib.SsbError, match="offsets"):
        enc(x, utt_offsets=[0, 1])
    with pytest.raises(ValueError):
        enc(np.zeros((2, 4, 41), np.float32))
    assert torch.equal(enc(x)["hidden"], enc(x)["hidden"])


def _voice(n, sr=16000, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    f0 = 160 + 60 * np.sin(2 * np.pi * 0.9 * t)
    y = sum(0.2 / k * np.sin(2 * np.pi * k * np.cumsum(f0) / sr) for k in range(1, 12))
    return (y * (0.6 + 0.4 * np.sin(2 * np.pi * 1.3 * t)) + 0.005 * rng.standard_normal(n)).astype(np.float32)


def test_emotion_mel_and_embed_utterance_match_the_oracle():
    from stylesinger_b200 import emotion
    g = np.load(GOLD)
    sd = FO.emotion_encoder_weights(int(g["seed"]))
    emotion.load_model({"model_state": {k: torch.from_numpy(v) for k, v in sd.items()}}, DEV)
    assert emotion.is_loaded()
    for n in (16000 * 6, 41234, 3000):
        y = _voice(n, seed=n)
        mel = emotion.wav_to_mel_spectrogram(y)
        ref = FO.emotion_mel(y)
        assert mel.shape == ref.shape == (1 + n // 160, 40)
        d = np.abs(mel - ref).max() / ref.max()
        print(f"n={n}: emotion mel max |d| / max {d:.3e}")
        assert d < 2e-5
        # embed_utterance: the reference's own composition (inference.py:110-155) of the restated pieces
        wav_sl, mel_sl = FO.compute_partial_slices(n)
        yp = np.pad(y, (0, max(0, wav_sl[-1][1] - n)))
        fr = FO.emotion_mel(yp)
        hid = FO.lstm_hidden(np.stack([fr[a:b] for a, b in mel_sl]), sd)
        emb, partials, wave_slices = emotion.embed_utterance(y, return_partials=True)
        du, dp = np.abs(emb - FO.utterance_embed(hid)).max(), np.abs(partials - hid).max()
        print(f"n={n}: {len(mel_sl)} partials, utterance embed {du:.3e}, partial hidden {dp:.3e}")
        assert emb.shape == (256,) and abs(np.linalg.norm(emb) - 1) < 1e-5 and du < 2e-6 and dp < 2e-6
        assert [(s.start, s.stop) for s in wave_slices] == wav_sl
        whole = emotion.embed_utterance(y, using_partials=False)
        assert np.abs(whole - FO.lstm_hidden(FO.emotion_mel(y)[None], sd)[0]).max() < 2e-6
