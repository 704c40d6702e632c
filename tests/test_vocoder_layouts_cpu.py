"""HiFi-GAN V2 and V3 without a GPU: the oracle's generator against the reference's own
HifiGanGenerator (tools/make_golden.py vocoder_layouts: 1-24 frames, with and without f0), its float64 mode against its
fp32 mode, synth's state-dict names against the reference's, and the config checks of ssb_vocoder_create_ex, which
refuse a layout before anything is allocated."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG, HIFIGAN_V2, HIFIGAN_V3
from tests.common import VOCODER_LAYOUTS, golden, vocoder_sd

TOL = 2e-6  # the reference bar of tests/test_vocoder_cpu.py
F64_BAR = 1e-5  # fp32 vs float64 oracle, as in tests/test_vocoder_cpu.py


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


@pytest.fixture(scope="module")
def fx():
    return golden("ref_vocoder_layouts")


def _cases(g, meta):
    """(layout, L, with_f0, mel, f0, seed, reference wav) of every stored reference run."""
    for name in meta["layouts"]:
        for L in meta["lengths"]:
            mel, f0 = g[f"mel_{L}"], g[f"f0_{L}"]
            if VOCODER_LAYOUTS[name]["use_pitch_embed"]:
                yield name, L, True, mel, f0, meta["seed"] + L, g[f"wav_{name}_{L}"]
            yield name, L, False, mel, None, meta["seed"] + L, g[f"wav_nof0_{name}_{L}"]


def test_fixture_covers_the_layouts(fx):
    g, meta = fx
    assert meta["layouts"] == ["v2", "v3", "v3_nonsf"] and meta["lengths"] == [1, 2, 3, 5, 17, 24]
    assert "wav_v3_nonsf_24" not in g.files  # the generator without NSF has no f0 input
    for L in meta["lengths"]:
        assert g[f"mel_{L}"].shape == (L, 80) and g[f"f0_{L}"].shape == (L,)
        for name, h in VOCODER_LAYOUTS.items():
            assert g[f"wav_nof0_{name}_{L}"].shape == (256 * L,)


@pytest.mark.parametrize("name", ["v2", "v3", "v3_nonsf"])
def test_oracle_matches_reference(fx, name):
    g, meta = fx
    worst = 0.0
    for lname, L, with_f0, mel, f0, seed, ref in _cases(g, meta):
        if lname != name:
            continue
        w = O.spec2wav(mel, f0, vocoder_sd(name), VOCODER_LAYOUTS[name], O.NoiseSource(seed))
        e = _maxabs(w, ref)
        print(f"{name} L={L:2d} f0={with_f0}: oracle vs reference max |d| {e:.2e} (bar {TOL:.0e})")
        assert w.shape == ref.shape
        worst = max(worst, e)
    assert worst < TOL


@pytest.mark.parametrize("name", ["v2", "v3", "v3_nonsf"])
def test_float64_oracle_agrees_with_fp32_oracle(fx, name):
    g, meta = fx
    worst = 0.0
    for lname, L, with_f0, mel, f0, seed, _ in _cases(g, meta):
        if lname != name:
            continue
        a = O.spec2wav(mel, f0, vocoder_sd(name), VOCODER_LAYOUTS[name], O.NoiseSource(seed))
        b = O.spec2wav(mel, f0, vocoder_sd(name), VOCODER_LAYOUTS[name], O.NoiseSource(seed), torch.float64)
        assert b.dtype == np.float64
        worst = max(worst, _maxabs(a, b))
    print(f"{name}: fp32 vs float64 oracle max |d| {worst:.2e} (bar {F64_BAR:.0e})")
    assert worst < F64_BAR


def test_synth_names_are_the_reference_names(fx):
    g, meta = fx
    for name in meta["layouts"]:
        assert [n for n, _ in synth.vocoder_param_shapes(VOCODER_LAYOUTS[name])] == meta["keys"][name], name
    assert any(".convs.1." in k for k in meta["keys"]["v3"]) and not any("convs1" in k for k in meta["keys"]["v3"])


def test_fixture_exercises_the_convs(fx):
    """tanh does not flatten the fixture: the waveforms vary and hardly any sample sits in saturation."""
    g, meta = fx
    for name, L, with_f0, *_, ref in _cases(g, meta):
        assert ref.std() > 1e-3, (name, L, with_f0)
        assert (np.abs(ref) > 0.999).mean() < 0.01, (name, L, with_f0)


# ---------------------------------------------------------------------------------------------------------------------
def _create_ex(h, **fields):
    """ssb_vocoder_create_ex on a config from h (fields override struct members) and an empty tensor list."""
    from stylesinger_b200._lib import TensorDesc, lib
    from stylesinger_b200.engine import vocoder_config_ex
    vc = vocoder_config_ex(h)
    for k, v in fields.items():
        if k == "res_dilations":
            for (j, m), d in v.items():
                vc.res_dilations[j][m] = d
        else:
            setattr(vc, k, v)
    arr = (TensorDesc * 1)()
    handle = C.c_void_p(12345)
    rc = lib.ssb_vocoder_create_ex(C.byref(handle), arr, 0, C.byref(vc))
    return rc, handle.value, lib.ssb_last_error().decode()


@pytest.mark.parametrize("h, fields, cause", [
    (HIFIGAN_V3, {"resblock": 3}, "resblock must be 1"),
    (HIFIGAN_V3, {"resblock": 0}, "resblock must be 1"),
    (DEFAULT_VOCODER_CONFIG, {"res_dilations": {(1, 2): 0}}, "is below 1"),
    (HIFIGAN_V3, {"res_dilations": {(2, 1): -2}}, "is below 1"),
    (HIFIGAN_V2, {"initial_channel": 96}, "multiple of 32, or 16 or 8"),  # stages of 48, 24, 12, 6 channels
    (HIFIGAN_V2, {"initial_channel": 64}, "multiple of 32, or 16 or 8"),  # last stage of 4 channels
    (HIFIGAN_V2, {"initial_channel": 100}, "multiple of 32, or 16 or 8"),  # 100 / 8 is not an integer
    # stage 2 (16 channels) at cumulative rate 1 * 1 * 2 = 2; stage 3 (8 channels) at 4 * 1 * 1 * 3 = 12
    (HIFIGAN_V2, {"up_rates": (C.c_int32 * 8)(1, 1, 2, 2)}, "not a multiple of 64 / 16"),
    (HIFIGAN_V2, {"up_rates": (C.c_int32 * 8)(4, 1, 1, 3)}, "not a multiple of 64 / 8"),
], ids=["resblock3", "resblock0", "dilation0_rb1", "dilation_neg_rb2", "c48", "c4", "c12.5", "rate_c16", "rate_c8"])
def test_create_ex_refuses_bad_layouts_without_a_gpu(h, fields, cause):
    rc, handle, err = _create_ex(h, **fields)
    print(f"{fields}: rc={rc}, {err}")
    assert rc != 0 and handle is None and cause in err


def test_create_ex_reads_only_the_dilations_of_its_resblock():
    """ResBlock2 reads two dilations per block: a zero in the third slot is not a refusal (the call then fails on the
    empty tensor list instead), while ResBlock1 refuses it."""
    rc, handle, err = _create_ex(HIFIGAN_V3, res_dilations={(0, 2): 0})
    assert rc != 0 and handle is None and "missing tensor" in err, err
    rc, handle, err = _create_ex(DEFAULT_VOCODER_CONFIG, res_dilations={(0, 2): 0})
    assert rc != 0 and handle is None and "is below 1" in err


def test_engine_config_refuses_short_dilation_lists():
    from stylesinger_b200.engine import vocoder_config_ex
    with pytest.raises(ValueError, match="reads 3 dilations"):
        vocoder_config_ex(dict(DEFAULT_VOCODER_CONFIG, resblock_dilation_sizes=[[1, 3], [1, 3], [1, 3]]))
    with pytest.raises(ValueError, match="reads 2 dilations"):
        vocoder_config_ex(dict(HIFIGAN_V3, resblock_dilation_sizes=[[1], [2], [3]]))
    with pytest.raises(ValueError, match="resblock must be"):
        vocoder_config_ex(dict(HIFIGAN_V3, resblock="3"))
    vc = vocoder_config_ex(dict(HIFIGAN_V3, resblock_dilation_sizes=[[1, 2, 9], [2, 6, 9], [3, 12, 9]]))
    assert vc.resblock == 2 and [list(vc.res_dilations[j])[:2] for j in range(3)] == [[1, 2], [2, 6], [3, 12]]
    assert all(vc.res_dilations[j][2] == 0 for j in range(3))  # the third entry is not passed
    assert vocoder_config_ex(DEFAULT_VOCODER_CONFIG).resblock == 1


# ---------------------------------------------------------------------------------------------------------------------
def _write_json_dir(d, gens):
    """A vocoder directory of the official HiFi-GAN release form: config.json + generator_v* ({'generator': sd})."""
    import json
    import os
    for fname, h in gens.items():
        torch.save({"generator": synth.vocoder_state_dict(h, seed=0)}, os.path.join(d, fname))
    with open(os.path.join(d, "config.json"), "w") as f:
        json.dump(list(gens.values())[0], f)


@pytest.mark.parametrize("fname, h", [("generator_v2", HIFIGAN_V2), ("generator_v3", HIFIGAN_V3)])
def test_load_vocoder_checkpoint_reads_v2_and_v3(tmp_path, fname, h):
    from stylesinger_b200 import formats
    _write_json_dir(str(tmp_path), {fname: h})
    sd, cfg, path = formats.load_vocoder_checkpoint(str(tmp_path))
    assert path.endswith(fname) and cfg["resblock"] == h["resblock"]
    assert list(sd) == [n for n, _ in synth.vocoder_param_shapes(h)]


def test_load_vocoder_checkpoint_prefers_v1_and_refuses_two_others(tmp_path):
    import os
    from stylesinger_b200 import formats
    a, b = tmp_path / "a", tmp_path / "b"
    a.mkdir()
    b.mkdir()
    _write_json_dir(str(a), {"generator_v1": DEFAULT_VOCODER_CONFIG, "generator_v3": HIFIGAN_V3})
    sd, cfg, path = formats.load_vocoder_checkpoint(str(a))
    assert os.path.basename(path) == "generator_v1" and any("convs1" in k for k in sd)
    _write_json_dir(str(b), {"generator_v2": HIFIGAN_V2, "generator_v3": HIFIGAN_V3})
    with pytest.raises(ValueError, match="generator_v2 and generator_v3"):
        formats.load_vocoder_checkpoint(str(b))
