"""HiFi-GAN V2 and V3 (ssb_vocoder_create_ex) on the tensor-core and the FFMA path: V2's 16- and 8-channel stages and
V3's 32-channel stage run their ResBlock convs as 64-channel convs over groups of 64 / C time steps, and V3's blocks are
ResBlock2.  Every check runs for V2, V3 and V3 without the NSF source:

  (a) against the reference's own generator (tests/golden/ref_vocoder_layouts.npz, noise injected as NoiseSource draws);
  (b) a ragged batch at the edge lengths of tests/test_gpu_vocoder.py and a bench-shaped batch against the float64
      oracle (pinned to the reference in tests/test_vocoder_layouts_cpu.py);
  (c) every utterance of a batch against its solo call;
  (d) with per-utterance seeds, utterance b against the B = 1 call with seeds[b];
  (e) which kernels run: with tensor cores on, every ResBlock conv (the grouped narrow ones included) and every eligible
      transposed conv launches on the tensor-core kernel; with them off, nothing does;
  (f) the workspace contract of tests/test_gpu_vocoder.py::test_workspace_contract;
and (g) V1 built through ssb_vocoder_create_ex gives the waveform and the kernel launches of ssb_vocoder_create.

Bars (max |d| on the tanh-bounded waveform) follow tests/test_gpu_vocoder.py: at most 4x the largest error measured on
an H100 SXM (80 GB, 700 W power limit) and at least 10x below the smallest miss of each of these deliberate bugs: the
grouped packing's input phase off by one, dilation d instead of d / g in the dilated grouped conv, ResBlock2's residual
taken from the block input instead of the running r, and conv_post reading the 8-channel stage with a stride of 16.
Each test prints what it measured; the measured errors and the bugs' misses are listed next to the bars.  A bug only
shows where its code runs: the grouped packing is tensor-core only at C = 32 (V3's grouped stage), ResBlock2 is V3's, and
the 8-channel conv_post is V2's.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG
from tests.common import VOCODER_LAYOUTS, golden, vocoder_sd

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HOP = 256
LAYOUTS = ["v2", "v3", "v3_nonsf"]
PATHS = [True, False]

# Measured max |d| over V2, V3 and V3 without NSF: tensor cores vs the float64 oracle or the reference 8.9e-6, FFMA 2.7e-6,
# tensor cores vs FFMA 9.0e-6, batch vs solo 3.2e-6 (tensor cores; bit-identical on FFMA and with keyed seeds).  The
# deliberate bugs missed the reference fixture or the edge-batch oracle by at least: input phase off by one 0.91 (V2, V3
# and V3 without NSF on tensor cores, V2 on FFMA), d instead of d / g 0.91 (V3 and V3 without NSF on tensor cores),
# ResBlock2 residual from the block input 0.87 (V3 and V3 without NSF, both paths), conv_post stride 16 1.2 (V2, both).
BAR_ORACLE = {True: 3.5e-5, False: 1e-5}  # CUDA (tensor cores / FFMA) vs float64 oracle or the reference
BAR_PATHS = 3.5e-5  # tensor-core path vs FFMA path of the same call
BAR_SOLO = 1.2e-5  # an utterance in a batch vs the same utterance alone

EDGE_LENGTHS = [160, 1, 17, 2, 33, 3, 16, 5, 15]
SHORT = [1, 3, 17, 64, 200]


def _offs(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def _synth_utt(L, seed):
    g = torch.Generator().manual_seed(seed)
    mel = (-3.0 + 1.0 * torch.randn(L, 80, generator=g)).clamp(-6, 1.5)
    f0 = 150 + 350 * torch.rand(L, generator=g)
    f0[: max(1, L // 10)] = 0
    for s in range(L // 3, L, 300):
        f0[s: s + 1 + L // 20] = 0
    return mel.numpy(), f0.numpy()


class Utt:
    """One utterance with the noise NoiseSource(seed) gives the oracle (see tests/test_gpu_vocoder.py)."""

    def __init__(self, mel, f0, seed):
        self.mel, self.f0, self.seed, self.L = mel, f0, seed, mel.shape[0]
        ns = O.NoiseSource(seed)
        self.ini = ns.rand((1, 9))[0]
        self.ini[0] = 0
        self.src = ns.randn((1, self.L * HOP, 9))[0]


def _cat(utts):
    mel = torch.from_numpy(np.concatenate([u.mel for u in utts])).to(DEV)
    f0 = torch.from_numpy(np.concatenate([u.f0 for u in utts])).to(DEV)
    ini = torch.stack([u.ini for u in utts]).contiguous().to(DEV)
    src = torch.cat([u.src for u in utts]).contiguous().to(DEV)
    return mel, f0, ini, src, _offs([u.L for u in utts])


def _generate(v, utts, with_f0=True):
    mel, f0, ini, src, offs = _cat(utts)
    if not with_f0:
        return v.generate(mel, None, offs).cpu().numpy()
    return v.generate(mel, f0, offs, rand_ini=ini, src_noise=src).cpu().numpy()


def _split(wav, utts):
    o = _offs([u.L for u in utts]) * HOP
    return [wav[o[i]:o[i + 1]] for i in range(len(utts))]


def _f0_modes(name):
    return (True, False) if VOCODER_LAYOUTS[name]["use_pitch_embed"] else (False,)


_V, _M = {}, {}


def _voc(name, tc):
    from stylesinger_b200.engine import Vocoder
    if name not in _V:
        _V[name] = Vocoder(vocoder_sd(name), VOCODER_LAYOUTS[name])
    v = _V[name]
    assert v.set_tensor_cores(tc) == tc
    return v


def _oracle(name, key, u, with_f0):
    k = (name, key, u.L, with_f0)
    if k not in _M:
        _M[k] = O.spec2wav(u.mel, u.f0 if with_f0 else None, vocoder_sd(name), VOCODER_LAYOUTS[name],
                           O.NoiseSource(u.seed), torch.float64)
    return _M[k]


def _report(name, errs, bars):
    for k, e in errs.items():
        print(f"{name}: {k} max |d| {e:.3e} (bar {bars[k]:.2g})")
    bad = {k: e for k, e in errs.items() if not e < bars[k]}
    assert not bad, bad


def _ids(tc):
    return "tc" if tc else "ffma"


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tc", PATHS, ids=_ids)
@pytest.mark.parametrize("name", LAYOUTS)
def test_matches_reference_fixture(name, tc):
    """(a) One ragged call of the fixture's six utterances (1-24 frames) against the reference's waveforms."""
    g, meta = golden("ref_vocoder_layouts")
    v = _voc(name, tc)
    utts = [Utt(g[f"mel_{L}"], g[f"f0_{L}"], meta["seed"] + L) for L in meta["lengths"]]
    worst = 0.0
    for with_f0 in _f0_modes(name):
        wav = _split(_generate(v, utts, with_f0), utts)
        for u, w in zip(utts, wav):
            ref = g[f"wav_{name}_{u.L}" if with_f0 else f"wav_nof0_{name}_{u.L}"]
            e = _maxabs(w, ref)
            print(f"  {name} L={u.L:2d} f0={with_f0}: vs reference {e:.2e}")
            worst = max(worst, e)
    _report(f"{name} {_ids(tc)} reference fixture", {"reference": worst}, {"reference": BAR_ORACLE[tc]})


def edge_utts():
    return [Utt(*_synth_utt(L, 500 + L), 600 + L) for L in EDGE_LENGTHS]


@pytest.mark.parametrize("tc", PATHS, ids=_ids)
@pytest.mark.parametrize("name", LAYOUTS)
def test_edge_batch_matches_float64_oracle_and_solo(name, tc):
    """(b, c) One ragged call of 1-160 frame utterances against the float64 oracle and against each solo call."""
    v = _voc(name, tc)
    utts = edge_utts()
    errs = {"oracle": 0.0, "solo": 0.0}
    for with_f0 in _f0_modes(name):
        wav = _split(_generate(v, utts, with_f0), utts)
        for u, w in zip(utts, wav):
            e = _maxabs(w, _oracle(name, "edge", u, with_f0))
            s = _maxabs(w, _generate(v, [u], with_f0))
            print(f"  {name} L={u.L:4d} f0={with_f0}: vs oracle {e:.2e}, vs solo {s:.2e}")
            errs["oracle"], errs["solo"] = max(errs["oracle"], e), max(errs["solo"], s)
    _report(f"{name} {_ids(tc)} edge batch", errs, {"oracle": BAR_ORACLE[tc], "solo": BAR_SOLO})


def bench_utts():
    """14 utterances, 21,384 frames (tests/test_gpu_vocoder.py::bench_utts): 9 long ones of the batch64 workload
    interleaved with 5 short ones."""
    fr = [int(round(187.5 * s)) for s in synth.batch_seconds(64, seed=1234)]
    longs = [f for f in fr if f >= 1800][:9]
    lens = []
    for i, L in enumerate(longs):
        lens.append(L)
        if i < len(SHORT):
            lens.append(SHORT[i])
    return [Utt(*_synth_utt(L, 700 + i), 800 + i) for i, L in enumerate(lens)]


@pytest.mark.parametrize("name", LAYOUTS)
def test_bench_shaped_call(name):
    """(b, c) The call size Vocoder.generate hands the library in the batch64 workload, on both paths: the short
    utterances against the float64 oracle, every utterance tensor cores vs FFMA and against its solo call."""
    utts = bench_utts()
    with_f0 = VOCODER_LAYOUTS[name]["use_pitch_embed"]
    w_tc = _split(_generate(_voc(name, True), utts, with_f0), utts)
    w_ffma = _split(_generate(_voc(name, False), utts, with_f0), utts)
    errs = {"oracle_tc": 0.0, "oracle_ffma": 0.0, "paths": 0.0, "solo_tc": 0.0, "solo_ffma": 0.0}
    for u, a, b in zip(utts, w_tc, w_ffma):
        p = _maxabs(a, b)
        s2 = _maxabs(b, _generate(_voc(name, False), [u], with_f0))
        s1 = _maxabs(a, _generate(_voc(name, True), [u], with_f0))
        line = f"  {name} L={u.L:5d}: tc vs ffma {p:.2e}, solo tc {s1:.2e}, solo ffma {s2:.2e}"
        if u.L in SHORT:
            ref = _oracle(name, "bench", u, with_f0)
            e1, e2 = _maxabs(a, ref), _maxabs(b, ref)
            errs["oracle_tc"], errs["oracle_ffma"] = max(errs["oracle_tc"], e1), max(errs["oracle_ffma"], e2)
            line += f", tc vs oracle {e1:.2e}, ffma vs oracle {e2:.2e}"
        print(line)
        errs["paths"] = max(errs["paths"], p)
        errs["solo_tc"], errs["solo_ffma"] = max(errs["solo_tc"], s1), max(errs["solo_ffma"], s2)
    _voc(name, True)
    _report(f"{name} bench-shaped call", errs, {"oracle_tc": BAR_ORACLE[True], "oracle_ffma": BAR_ORACLE[False],
                                                "paths": BAR_PATHS, "solo_tc": BAR_SOLO, "solo_ffma": BAR_SOLO})


@pytest.mark.parametrize("tc", PATHS, ids=_ids)
@pytest.mark.parametrize("name", LAYOUTS)
def test_keyed_seeds_match_solo_calls(name, tc):
    """(d) ssb_hifigan_generate_keyed: utterance b of a batch is the B = 1 call with seeds[b]."""
    v = _voc(name, tc)
    utts = edge_utts()
    mel, f0, _, _, offs = _cat(utts)
    f0 = f0 if VOCODER_LAYOUTS[name]["use_pitch_embed"] else None
    seeds = [1000003 * (b + 1) + 17 for b in range(len(utts))]
    wav = v.generate(mel, f0, offs, seeds=seeds).cpu().numpy()
    worst = 0.0
    for b in range(len(utts)):
        a, e = int(offs[b]), int(offs[b + 1])
        w = v.generate(mel[a:e], None if f0 is None else f0[a:e], np.array([0, e - a], np.int32), seeds=[seeds[b]])
        worst = max(worst, _maxabs(wav[a * HOP:e * HOP], w.cpu().numpy()))
    _report(f"{name} {_ids(tc)} keyed seeds", {"solo": worst}, {"solo": BAR_SOLO})


def _expected_tc_launches(h):
    """Tensor-core GEMMs of one call: every ResBlock conv (C % 64 == 0 or grouped: all of them) and each transposed conv
    whose Cin and N = u * C are multiples of 64."""
    n = 0
    nconv = 6 if str(h["resblock"]) == "1" else 2
    for i, u in enumerate(h["upsample_rates"]):
        c = h["upsample_initial_channel"] // 2 ** (i + 1)
        n += len(h["resblock_kernel_sizes"]) * nconv
        n += 1 if (2 * c) % 64 == 0 and (u * c) % 64 == 0 else 0
    return n


@pytest.mark.parametrize("name", LAYOUTS)
def test_variant_counts(name):
    """(e) With tensor cores on, the narrow stages' grouped ResBlock convs run on the tensor-core kernel (the count of
    tensor-core launches is that of every ResBlock conv plus the eligible transposed convs); with them off, none do."""
    from stylesinger_b200._lib import variant_launches
    utts = edge_utts()[:3]
    counts = {}
    for tc in PATHS:
        v = _voc(name, tc)
        torch.cuda.synchronize()
        before = variant_launches()
        _generate(v, utts, VOCODER_LAYOUTS[name]["use_pitch_embed"])
        after = variant_launches()
        counts[tc] = sum(after[k] - before.get(k, 0) for k in after)
    exp = _expected_tc_launches(VOCODER_LAYOUTS[name])
    print(f"{name}: tensor-core launches with tensor cores on {counts[True]} (expected {exp}), off {counts[False]}")
    _voc(name, True)
    assert counts[True] == exp and counts[False] == 0


# ---------------------------------------------------------------------------------------------------------------------
TAIL = 1 << 20


def _raw_generate(v, utts, ws, ws_bytes, with_f0):
    from stylesinger_b200._lib import check, lib
    mel, f0, ini, src, offs = _cat(utts)
    wav = torch.empty(int(offs[-1]) * HOP, dtype=torch.float32, device=DEV)
    p = lambda t: C.c_void_p(t.data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.ssb_hifigan_generate(v._h, p(mel), p(f0) if with_f0 else None, offs.ctypes.data, len(utts),
                                   p(ini) if with_f0 else None, p(src) if with_f0 else None, 0, p(wav), p(ws), ws_bytes,
                                   stream), "ssb_hifigan_generate")
    torch.cuda.synchronize()
    return wav


def _ws_bytes(v, utts):
    from stylesinger_b200._lib import lib
    offs = _offs([u.L for u in utts])
    n = int(lib.ssb_vocoder_workspace_bytes(v._h, offs.ctypes.data, len(utts)))
    assert n > 0
    return n


@pytest.mark.parametrize("tc", PATHS, ids=_ids)
@pytest.mark.parametrize("name", LAYOUTS)
def test_workspace_contract(name, tc):
    """(f) ssb_vocoder_workspace_bytes is enough, the call reads no byte it has not written (0xFF and zeroed workspaces
    give the same bits), writes nothing past that size (a sentinel tail survives), and a workspace left over from a
    larger call of another shape changes nothing."""
    v = _voc(name, tc)
    with_f0 = VOCODER_LAYOUTS[name]["use_pitch_embed"]
    big, small = bench_utts()[:6], edge_utts()
    nb, ns = _ws_bytes(v, big), _ws_bytes(v, small)
    print(f"{name} {_ids(tc)} workspace bytes: bench-shaped call {nb}, edge batch {ns}")
    g = torch.Generator(device=DEV).manual_seed(5)
    sentinel = torch.randint(0, 256, (TAIL,), generator=g, device=DEV, dtype=torch.int32).to(torch.uint8)
    try:
        ws = torch.empty(nb + TAIL, dtype=torch.uint8, device=DEV)
        ws[nb:] = sentinel
        ws[:nb].fill_(0xFF)
        a = _raw_generate(v, big, ws, nb, with_f0)
        assert torch.equal(ws[nb:], sentinel), "the call wrote past ssb_vocoder_workspace_bytes"
        ws[:nb].zero_()
        b = _raw_generate(v, big, ws, nb, with_f0)
        assert torch.equal(ws[nb:], sentinel)
        assert torch.isfinite(a).all() and torch.equal(a, b), "the result depends on workspace bytes the call never wrote"
        c = _raw_generate(v, small, ws, nb, with_f0)
        del ws
        ws2 = torch.zeros(ns + TAIL, dtype=torch.uint8, device=DEV)
        ws2[ns:] = sentinel
        d = _raw_generate(v, small, ws2, ns, with_f0)
        ws2[:ns].fill_(0xFF)
        e = _raw_generate(v, small, ws2, ns, with_f0)
        assert torch.equal(ws2[ns:], sentinel), "the edge batch wrote past ssb_vocoder_workspace_bytes"
        assert torch.isfinite(c).all() and torch.equal(c, d) and torch.equal(d, e)
    finally:
        _voc(name, True)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tc", PATHS, ids=_ids)
def test_v1_through_create_ex_is_bit_identical(tc):
    """(g) ssb_vocoder_create is ssb_vocoder_create_ex with resblock = 1: V1 built either way gives the same waveform,
    bit for bit, and launches the same tensor-core kernel variants the same number of times."""
    from stylesinger_b200._lib import TensorDesc, VocoderConfig, check, lib, variant_launches
    from stylesinger_b200.engine import Vocoder, _descs, vocoder_config_ex
    sd = vocoder_sd()
    v_ex = Vocoder(sd, DEFAULT_VOCODER_CONFIG)
    v_old = Vocoder(sd, DEFAULT_VOCODER_CONFIG)
    ex = vocoder_config_ex(DEFAULT_VOCODER_CONFIG)
    vc = VocoderConfig()
    for f, _ in VocoderConfig._fields_:
        setattr(vc, f, getattr(ex, f))
    tensors = {k: t for k, t in sd.items() if isinstance(t, torch.Tensor)}
    arr, keep = _descs(tensors)
    h = C.c_void_p()
    check(lib.ssb_vocoder_create(C.byref(h), arr, len(tensors), C.byref(vc)), "ssb_vocoder_create")
    lib.ssb_vocoder_free(v_old._h)
    v_old._h = h
    utts = edge_utts()[:5] + bench_utts()[:2]
    out, launches = {}, {}
    for key, v in (("ex", v_ex), ("old", v_old)):
        v.set_tensor_cores(tc)
        torch.cuda.synchronize()
        before = variant_launches()
        out[key] = _generate(v, utts)
        after = variant_launches()
        launches[key] = {k: after[k] - before.get(k, 0) for k in after if after[k] != before.get(k, 0)}
    print(f"V1 {_ids(tc)}: launches through create_ex {launches['ex']}, through create {launches['old']}")
    assert np.array_equal(out["ex"], out["old"])
    assert launches["ex"] == launches["old"]


@pytest.mark.parametrize("fname, name", [("generator_v1", None), ("generator_v2", "v2"), ("generator_v3", "v3")])
def test_checkpoint_directory_to_waveform(tmp_path, fname, name):
    """A config.json + generator_v* directory goes through formats.load_vocoder_checkpoint into engine.Vocoder and gives
    the waveform of the same weights built directly."""
    import json
    from stylesinger_b200 import formats
    from stylesinger_b200.engine import Vocoder
    h = DEFAULT_VOCODER_CONFIG if name is None else VOCODER_LAYOUTS[name]
    sd = vocoder_sd(name)
    torch.save({"generator": sd}, str(tmp_path / fname))
    with open(tmp_path / "config.json", "w") as f:
        json.dump(h, f)
    vsd, cfg, path = formats.load_vocoder_checkpoint(str(tmp_path))
    assert path.endswith(fname)
    utts = edge_utts()[:4]
    a = _generate(Vocoder(vsd, cfg), utts)
    b = _generate(Vocoder(sd, h), utts)
    print(f"{fname}: {a.size} samples, max |wav| {np.abs(a).max():.3f}")
    assert np.isfinite(a).all() and np.abs(a).max() > 1e-2 and np.array_equal(a, b)
