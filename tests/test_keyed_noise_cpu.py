"""Per-utterance Philox seeds without a GPU: the argument checks of every Python entry that takes `seeds`, the NumPy keyed
draw plan (tests/keyed_plan.py) against the per-call plan of tests/philox_ref.py, and the seeds of
tools/infer_dataset.py --seed-per-item."""
import importlib.util
import os
import types

import numpy as np
import pytest
import torch

from stylesinger_b200.engine import AcousticModel, PackedBatch, Vocoder, utt_seeds
from stylesinger_b200.infer import StyleSingerInfer
from stylesinger_b200.modules import StyleSinger
from tests import keyed_plan as K
from tests import philox_ref as P

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- argument checks ---------------------------------------------------------------------------------------------------
def test_utt_seeds_accepts_the_full_64_bit_range():
    s = utt_seeds([0, 1, 2**63, 2**64 - 1, np.uint64(7), np.int64(9)], 6)
    assert s.dtype == np.uint64 and s.tolist() == [0, 1, 2**63, 2**64 - 1, 7, 9]


@pytest.mark.parametrize("seeds,B,exc", [
    ([1, 2], 3, ValueError),            # one seed short
    ([1, 2, 3, 4], 3, ValueError),      # one too many
    ([1, -1, 2], 3, ValueError),        # below 0
    ([1, 2**64, 2], 3, ValueError),     # 2**64 does not fit
    ([1, 2.0, 3], 3, TypeError),        # not an integer
])
def test_utt_seeds_rejects(seeds, B, exc):
    with pytest.raises(exc):
        utt_seeds(seeds, B)


def _pb(B):
    fo = np.arange(B + 1, dtype=np.int32) * 5
    return PackedBatch(B=B, ph_offsets=fo, ref_offsets=fo, frame_offsets=fo, t={})


def _no_cuda(*a, **k):
    raise AssertionError("the argument check must fail before anything reaches the device")


def _stubs():
    """Objects that fail loudly if the entries go past their argument checks."""
    model = types.SimpleNamespace(_inputs=_no_cuda, _h=None, device="cuda:0")
    voc = types.SimpleNamespace(denoise_c=0.0, _h=None, _ws=None, device="cuda:0", hop=256, max_frames_per_call=24000)
    return model, voc


@pytest.mark.parametrize("seeds,noise", [
    ([1, 2], None),                              # wrong length
    ([1, 2, 2**64], None),                       # out of range
    ([1, 2, 3], {"mel": object()}),              # with injected mel noise
    ([1, 2, 3], {"f0_gauss": [object(), object()], "f0_unif": [object(), object()]}),
])
def test_acoustic_forward_checks_seeds_first(seeds, noise):
    model, _ = _stubs()
    with pytest.raises(ValueError):
        AcousticModel.forward(model, _pb(3), noise=noise, seeds=seeds)


@pytest.mark.parametrize("seeds,kw", [
    ([1], {}),
    ([1, -3], {}),
    ([1, 2], {"rand_ini": object()}),
    ([1, 2], {"src_noise": object()}),
])
def test_vocoder_generate_checks_seeds_first(seeds, kw):
    _, voc = _stubs()
    with pytest.raises(ValueError):
        Vocoder.generate(voc, None, None, np.array([0, 3, 7], np.int32), seeds=seeds, **kw)


def test_infer_entries_check_seeds_first():
    stub = types.SimpleNamespace(model=types.SimpleNamespace(predict_durations=_no_cuda, forward=_no_cuda),
                                 vocoder=types.SimpleNamespace(generate=_no_cuda), device="cuda:0")
    with pytest.raises(ValueError):
        StyleSingerInfer.infer_batch(stub, [{}, {}], seeds=[1])
    with pytest.raises(ValueError):
        StyleSingerInfer.infer_packed(stub, _pb(2), seeds=[1, 2**64])
    with pytest.raises(ValueError):
        StyleSingerInfer.run_device(stub, _pb(2), seeds=[1, 2], noise={"mel": object()})
    with pytest.raises(ValueError):
        StyleSingerInfer.run_device(stub, _pb(2), seeds=[1, 2], voc_noise={"rand_ini": object()})


def test_modules_facade_checks_seeds_first():
    stub = types.SimpleNamespace(hparams={}, engine=types.SimpleNamespace(forward=_no_cuda, predict_durations=_no_cuda))
    tok = torch.zeros(2, 4, dtype=torch.long)
    with pytest.raises(ValueError):
        StyleSinger.forward(stub, tok, infer=True, seeds=[1, 2, 3])
    with pytest.raises(ValueError):
        StyleSinger.forward(stub, tok, infer=True, seeds=[1, 2], noise={"mel": object()})


# ---- the keyed draw plan -----------------------------------------------------------------------------------------------
def test_keyed_plan_of_one_utterance_is_the_per_call_plan():
    """B = 1: the keyed plan with seeds [s] is, element for element, the per-call plan with seed s."""
    s, T, fo = 0xDEADBEEF0123, 3, np.array([0, 137])
    want = P.acoustic_noise(s, T, T, fo)
    got = K.acoustic_noise([s], T, T, fo)
    assert np.array_equal(got["mel"], want["mel"])
    for n in range(2):
        assert np.array_equal(got["f0_gauss"][n], want["f0_gauss"][n])
        assert np.array_equal(got["f0_unif"][n], want["f0_unif"][n])
    assert np.array_equal(K.vocoder_rand_ini([s]), P.vocoder_rand_ini(s, 1))
    assert np.array_equal(K.vocoder_src_noise([s], [0, 3], hop=16), P.vocoder_src_noise(s, [0, 3], hop=16))


def test_keyed_plan_gives_each_utterance_its_solo_draws():
    """Every utterance's rows of a keyed batch are its B = 1 draws, whatever its neighbours; the per-call plan of the same
    batch is not (its rows are counted through the whole call)."""
    lens, seeds, T = [5, 1, 130, 17], [11, 2**64 - 1, 0, 11], 2
    fo = np.concatenate([[0], np.cumsum(lens)])
    mel = K.mel_noise(seeds, T, fo)
    unif = K.f0_unif_noise(seeds, 1, T, fo)
    src = K.vocoder_src_noise(seeds, fo, hop=8)
    for b, n in enumerate(lens):
        a, e = fo[b], fo[b + 1]
        assert np.array_equal(mel[:, a:e], P.mel_noise(seeds[b], T, [0, n]))
        assert np.array_equal(unif[:, a:e], P.f0_unif_noise(seeds[b], 1, T, [0, n]))
        assert np.array_equal(src[a * 8:e * 8], P.vocoder_src_noise(seeds[b], [0, n], hop=8))
    # the same seed on two utterances of the batch (b = 0 and 3) gives them the same leading draws
    assert np.array_equal(mel[:, 0:5], mel[:, fo[3]:fo[3] + 5])
    legacy = P.mel_noise(seeds[0], T, fo)
    assert not np.array_equal(legacy[:, fo[3]:fo[3] + 5], mel[:, fo[3]:fo[3] + 5])


def test_keyed_rand_ini_reads_stream_zero_under_each_key():
    seeds = [3, 4, 3]
    r = K.vocoder_rand_ini(seeds)
    assert np.array_equal(r[0], r[2]) and not np.array_equal(r[0], r[1])
    assert np.array_equal(r[1], P.vocoder_rand_ini(4, 1)[0])


# ---- tools/infer_dataset.py --seed-per-item ------------------------------------------------------------------------------
def _tool():
    spec = importlib.util.spec_from_file_location("infer_dataset", os.path.join(REPO, "tools", "infer_dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_seed_per_item_is_the_seed_plus_the_dataset_index():
    tool = _tool()
    assert tool.item_seeds(100, [4, 0, 9]) == [104, 100, 109]
    # length-sorted order cut into batches of any size: each item keeps its seed
    order = [7, 2, 5, 0, 3]
    for b in (1, 2, 5):
        got = {}
        for i in range(0, len(order), b):
            got.update(zip(order[i:i + b], tool.item_seeds(5, order[i:i + b])))
        assert got == {i: 5 + i for i in order}
