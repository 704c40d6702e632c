"""Convolutional F0 generator (hparams['f0_gen'] == 'conv'), CPU side: the test oracle and the synthetic
checkpoint against the unmodified reference (tests/golden/ref_convf0.npz), the hparams rules, and the C ABI's argument
check (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from stylesinger_b200.hparams import resolve
from tests.common import conv_hp, conv_sd, golden, hp_for, predictor_inputs, utt_from_meta

TOL = 2e-5  # fp32 CPU, same op order up to BLAS blocking (as tests/test_oracle_golden.py)


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def _forward(meta, seed, use_mel2ph=True):
    u = utt_from_meta(meta)
    ns = O.NoiseSource(seed)
    with torch.no_grad():
        r = O.stylesinger_forward(conv_sd(meta), conv_hp(meta), u["txt_tokens"][None], u["note"][None],
                                  u["note_dur"][None], u["note_type"][None], u["spk_embed"][None],
                                  u["emo_embed"][None], u["ref_mels"][None], u["ref_f0"], ns,
                                  mel2ph=u["mel2ph"][None] if use_mel2ph else None)
    return r, ns


def _check_pitch(r, pitch_pred, f0_denorm, tag):
    """pitch_pred within TOL; uv (pitch_pred[..., 1] > 0) and the coarse bins exact."""
    e_pp = _maxabs(r["pitch_pred"][0].numpy(), pitch_pred)
    e_f0 = _maxabs(r["f0_denorm"][0].numpy(), f0_denorm)
    print(tag, "pitch_pred", e_pp, "f0_denorm(Hz)", e_f0)
    assert e_pp < TOL
    assert e_f0 < 1e-3
    assert np.array_equal(r["pitch_pred"][0, :, 1].numpy() > 0, pitch_pred[:, 1] > 0)
    assert np.array_equal(r["pitch"][0].numpy(), O.f0_to_coarse(torch.from_numpy(f0_denorm)).numpy())


def test_fixture_exercises_the_quantiser_and_both_uv_classes():
    """The synthetic f0 rows put the predicted pitch in the singing range: many distinct coarse bins, and both uv
    classes, as the fixture shows."""
    g, meta = golden("ref_convf0")
    for k in ("pitch_pred", "dur_pitch_pred", "pd_pitch_pred"):
        uv = g[k][:, 1] > 0
        assert 0.2 < uv.mean() < 0.8, k
    bins = O.f0_to_coarse(torch.from_numpy(g["f0_denorm"])).numpy()
    assert len(np.unique(bins[bins > 1])) >= 10
    assert 7.0 < g["pitch_pred"][:, 0].min() and g["pitch_pred"][:, 0].max() < 9.5


def test_oracle_predictors_match_reference():
    g, meta = golden("ref_convf0")
    xs = predictor_inputs(meta)
    assert np.array_equal(xs[:, :4].numpy(), g["pred_x_head"])  # the regenerated inputs are the reference's
    assert (xs[:, meta["pred_zero_rows"], 0] == 0).all()
    sd = conv_sd(meta)
    with torch.no_grad():
        for which, key in ((0, "pred_out_agnostic"), (1, "pred_out_specific")):
            out = O.pitch_predictor(xs[which][None], sd, which)[0]
            err = _maxabs(out.numpy(), g[key])
            print(key, "L-inf", err)
            assert err < TOL, (key, err)


def test_oracle_forward_matches_reference():
    g, meta = golden("ref_convf0")
    r, ns = _forward(meta, meta["seed"])
    assert [[k, list(sh)] for k, sh in ns.log] == meta["noise_log"]  # only the mel sampler draws
    assert all(list(sh) == [1, 1, 80, meta["frames"]] for _, sh in ns.log)
    _check_pitch(r, g["pitch_pred"], g["f0_denorm"], "mel2ph given:")
    for k in ("decoder_inp", "mel_out"):
        assert _maxabs(r[k][0].numpy(), g[k]) < TOL, k


def test_oracle_duration_path_matches_reference():
    g, meta = golden("ref_convf0")
    r, ns = _forward(meta, meta["seed"] + 1, use_mel2ph=False)
    assert [[k, list(sh)] for k, sh in ns.log] == meta["dur_noise_log"]
    assert np.array_equal(r["mel2ph"][0].numpy(), g["dur_mel2ph"])
    _check_pitch(r, g["dur_pitch_pred"], g["dur_f0_denorm"], "durations predicted:")
    assert _maxabs(r["decoder_inp"][0].numpy(), g["dur_decoder_inp"]) < TOL
    assert _maxabs(r["mel_out"][0].numpy(), g["dur_mel_out"]) < TOL


def test_oracle_prodiff_with_conv_f0_matches_reference():
    g, meta = golden("ref_convf0")
    pm = meta["prodiff"]
    r, ns = _forward(pm, pm["seed"])
    assert [[k, list(sh)] for k, sh in ns.log] == pm["noise_log"]
    _check_pitch(r, g["pd_pitch_pred"], g["pd_f0_denorm"], "ProDiff decoder:")
    assert _maxabs(r["decoder_inp"][0].numpy(), g["pd_decoder_inp"]) < TOL
    err, scale = _maxabs(r["mel_out"][0].numpy(), g["pd_mel_out"]), float(np.abs(g["pd_mel_out"]).max())
    assert err < TOL * max(1.0, scale), (err, scale)


def test_synth_conv_state_dicts_have_the_reference_keys_and_shapes():
    g, meta = golden("ref_convf0")
    for m in (meta, meta["prodiff"]):
        sd = conv_sd(m)
        assert [[k, list(v.shape)] for k, v in sd.items()] == m["state_dict"]
        assert not any(k.startswith(("gm_diffnet", "f0_gen")) for k in sd)
        assert sum(k.startswith("pitch_inpainter_predictor.") for k in sd) == 24


def test_synth_gmdiff_state_dict_is_unchanged_by_the_conv_rules():
    """The conv rules touch nothing a gmdiff checkpoint draws: every tensor the two configurations share before the
    first key that only one of them has is bit-identical, apart from the two f0 rows that the conv rule rescales."""
    gm = synth.acoustic_state_dict(hp_for(4), seed=0)
    cv = synth.acoustic_state_dict(resolve(timesteps=4, K_step=4, f0_gen="conv"), seed=0)
    assert not any(k.startswith("pitch_inpainter_predictor.") for k in gm)
    shared = 0
    for (kg, tg), (kc, tc) in zip(gm.items(), cv.items()):
        if kg != kc:
            assert kc.startswith("pitch_inpainter_predictor.") and kg.startswith("gm_diffnet.")
            break
        if kg in ("pitch_predictor.linear.weight", "pitch_predictor.linear.bias"):
            assert torch.equal(tg[1], tc[1])  # the uv row is left as generated
            continue
        assert torch.equal(tg, tc), kg
        shared += 1
    assert shared > 250
    assert float(cv["pitch_predictor.linear.bias"][0]) == 8.0
    assert torch.equal(cv["pitch_predictor.linear.weight"][0], gm["pitch_predictor.linear.weight"][0] * 0.35)


def test_resolve_accepts_conv_and_refuses_other_f0_generators():
    hp = resolve(f0_gen="conv")
    assert hp["f0_gen"] == "conv" and hp["predictor_kernel"] == 5
    assert resolve(f0_gen="conv", decoder="prodiff", schedule_type="vpsde")["f0_gen"] == "conv"
    for bad in ("diff", "CONV", None, "gmdiff2"):
        with pytest.raises(NotImplementedError):
            resolve(f0_gen=bad)


def test_model_create_ex2_rejects_an_unknown_f0_gen_without_a_gpu():
    from stylesinger_b200._lib import HParams, lib
    for mel_decoder, f0_gen, msg in ((0, 7, "unknown f0_gen 7"), (0, -1, "unknown f0_gen -1"),
                                     (5, 1, "unknown mel_decoder 5")):
        h = C.c_void_p()
        rc = lib.ssb_model_create_ex2(C.byref(h), None, 0, C.byref(HParams()), mel_decoder, f0_gen)
        err = lib.ssb_last_error().decode()
        print("rc", rc, "message:", err)
        assert rc != 0 and not h.value
        assert msg in err
