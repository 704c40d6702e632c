"""The HiFi-GAN-NSF vocoder (ssb_hifigan_generate) against the float64 oracle on bench-sized ragged batches and at
utterance-length edges, on the tensor-core and the FFMA path.

Every call injects its noise (rand_ini, src_noise), drawn per utterance exactly as the oracle draws it from
NoiseSource(seed), so every utterance of a batch has B = 1 semantics and can be checked against the oracle, against its
own solo call and against the other path.  The float64 oracle runs the conv stack in double precision (the NSF source
stays fp32, as in the reference and in k_nsf_phase); its own agreement with the reference is pinned in
tests/test_vocoder_cpu.py.

Bars (max |d| on the waveform, which tanh bounds to [-1, 1]) were set from errors measured on an H100 SXM (80 GB, 700 W
power limit): at most 4x the largest measured error and at least 10x below the smallest miss of each of these deliberate
bugs: the d = -1 / +1 taps of the transposed-conv packing swapped, gamma applied at every MRF branch, the NSF source
window of the tiled noise conv shifted by one sample at a block edge, the phase scan's carry not advanced across chunks,
a GEMM epilogue writing one row past the tile's valid rows (into a guard row), and Vocoder.generate slicing rand_ini one
group off.  Each test prints what it measured.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG
from tests.common import golden, vocoder_sd

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HOP = 256

# measured max |d|: tensor cores vs oracle 2.8e-5, FFMA vs oracle 3.5e-6, tensor cores vs FFMA 2.8e-5, solo 5.6e-6;
# FFMA vs oracle on the 10 s utterance 3.4e-6, and 1.0e-4 with the phase scan's carry broken
BAR_ORACLE = {True: 8e-5, False: 1.2e-5}  # CUDA (tensor cores / FFMA) vs float64 oracle
BAR_PATHS = 1e-4  # tensor-core path vs FFMA path of the same call
BAR_SOLO = 2e-5  # an utterance in a batch vs the same utterance alone (the batch size may select another kernel variant)
BAR_PHASE = 1e-5  # FFMA vs float64 oracle on the 10 s utterance (see test_nsf_phase_over_a_10s_utterance)

EDGE_LENGTHS = [160, 1, 17, 2, 33, 3, 16, 5, 15]  # below conv_pre's reach (1-3), around 16-frame tiles, odd and even
SHORT = [1, 3, 17, 64, 200]


def _offs(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def _synth_utt(L, seed):
    """mel with values at both clip bounds, f0 with unvoiced runs (a leading one, and one per ~300 frames)."""
    g = torch.Generator().manual_seed(seed)
    mel = (-3.0 + 2.0 * torch.randn(L, 80, generator=g)).clamp(-6, 1.5)
    f0 = 150 + 350 * torch.rand(L, generator=g)
    f0[: max(1, L // 10)] = 0
    for s in range(L // 3, L, 300):
        f0[s: s + 1 + L // 20] = 0
    return mel.numpy(), f0.numpy()


class Utt:
    """One utterance with the noise NoiseSource(seed) gives the oracle: rand_ini [9] (harmonic 0 zeroed, as the
    reference does) and src_noise [L * HOP, 9]."""

    def __init__(self, mel, f0, seed):
        self.mel, self.f0, self.seed, self.L = mel, f0, seed, mel.shape[0]
        ns = O.NoiseSource(seed)
        self.ini = ns.rand((1, 9))[0]
        self.ini[0] = 0
        self.src = ns.randn((1, self.L * HOP, 9))[0]

    def oracle(self, with_f0=True):
        with torch.no_grad():
            return O.spec2wav(self.mel, self.f0 if with_f0 else None, vocoder_sd(), DEFAULT_VOCODER_CONFIG,
                              O.NoiseSource(self.seed), torch.float64)


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


_M = {}


@pytest.fixture(scope="module")
def voc():
    from stylesinger_b200.engine import Vocoder
    v = Vocoder(vocoder_sd(), DEFAULT_VOCODER_CONFIG)
    yield v
    v.set_tensor_cores(True)


def _oracle(key, u, with_f0=True):
    k = (key, with_f0)
    if k not in _M:
        _M[k] = u.oracle(with_f0)
    return _M[k]


def edge_utts():
    g, meta = golden("ref_vocoder_edges")  # the reference's own edge inputs (voiced / unvoiced alternation, ~1100 Hz)
    utts = []
    for L in EDGE_LENGTHS:
        if L in meta["lengths"]:
            utts.append(Utt(g[f"mel_{L}"], g[f"f0_{L}"], meta["seed"] + L))
        else:
            utts.append(Utt(*_synth_utt(L, 500 + L), 600 + L))
    return utts


def _report(name, errs, bars):
    for k, e in errs.items():
        print(f"{name}: {k} max |d| {e:.3e} (bar {bars[k]:.2g})")
    bad = {k: e for k, e in errs.items() if not e < bars[k]}
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "ffma"])
def test_edge_batch_matches_float64_oracle_and_solo(voc, tc):
    """One ragged call of 1-160 frame utterances (partial 128-row tiles at stage 0 for lengths not a multiple of 16, at
    stage 1 for odd lengths; utterances shorter than conv_pre's reach), with and without f0."""
    voc.set_tensor_cores(tc)
    utts = edge_utts()
    errs = {"oracle": 0.0, "solo": 0.0}
    for with_f0 in (True, False):
        wav = _split(_generate(voc, utts, with_f0), utts)
        for u, w in zip(utts, wav):
            ref = _oracle(("edge", u.L), u, with_f0)
            e = _maxabs(w, ref)
            s = _maxabs(w, _generate(voc, [u], with_f0))
            print(f"  L={u.L:4d} f0={with_f0}: vs oracle {e:.2e}, vs solo {s:.2e}")
            errs["oracle"], errs["solo"] = max(errs["oracle"], e), max(errs["solo"], s)
    _report(f"edge batch {'tc' if tc else 'ffma'}", errs, {"oracle": BAR_ORACLE[tc], "solo": BAR_SOLO})


def bench_utts():
    """14 utterances, 21,384 frames: 9 long ones of the batch64 workload interleaved with 5 short ones."""
    fr = [int(round(187.5 * s)) for s in synth.batch_seconds(64, seed=1234)]
    longs = [f for f in fr if f >= 1800][:9]
    lens = []
    for i, L in enumerate(longs):
        lens.append(L)
        if i < len(SHORT):
            lens.append(SHORT[i])
    assert len(lens) == 14 and 20000 <= sum(lens) <= 24000
    return [Utt(*_synth_utt(L, 700 + i), 800 + i) for i, L in enumerate(lens)]


def test_bench_shaped_call(voc):
    """One call of the size Vocoder.generate hands the library in the batch64 workload: the CTA-pair GEMM variants run
    over a tile table with an utterance boundary every few hundred tiles, and the time-paired C = 32 stage at scale."""
    from stylesinger_b200._lib import variant_launches
    utts = bench_utts()
    voc.set_tensor_cores(True)
    before = variant_launches()
    w_tc = _split(_generate(voc, utts), utts)
    after = variant_launches()
    pair = {k: after[k] - before.get(k, 0) for k in after if k.startswith("tc2") and after[k] > before.get(k, 0)}
    print("CTA-pair variants launched:", pair)
    assert pair, "the bench-sized call ran no CTA-pair (tc2...) variant"
    voc.set_tensor_cores(False)
    w_ffma = _split(_generate(voc, utts), utts)
    voc.set_tensor_cores(True)
    errs = {"oracle_tc": 0.0, "oracle_ffma": 0.0, "paths": 0.0, "solo": 0.0}
    for u, a, b in zip(utts, w_tc, w_ffma):
        p, s = _maxabs(a, b), _maxabs(a, _generate(voc, [u]))
        line = f"  L={u.L:5d}: tc vs ffma {p:.2e}, vs solo {s:.2e}"
        if u.L in SHORT:
            ref = _oracle(("bench", u.L), u)
            e1, e2 = _maxabs(a, ref), _maxabs(b, ref)
            errs["oracle_tc"], errs["oracle_ffma"] = max(errs["oracle_tc"], e1), max(errs["oracle_ffma"], e2)
            line += f", tc vs oracle {e1:.2e}, ffma vs oracle {e2:.2e}"
        print(line)
        errs["paths"], errs["solo"] = max(errs["paths"], p), max(errs["solo"], s)
    _report("bench-shaped call", errs, {"oracle_tc": BAR_ORACLE[True], "oracle_ffma": BAR_ORACLE[False],
                                        "paths": BAR_PATHS, "solo": BAR_SOLO})


def test_nsf_phase_over_a_10s_utterance(voc):
    """k_nsf_phase carries its double-precision scan across 256-sample chunks and reproduces the reference's fp32 cumsum
    rounding.  A wrong wrap count only moves the phase by whole turns, so it shows as the fp32 rounding of a phase that
    grows by about one turn per chunk: invisible on short utterances, largest at the end of a long one.  One 1,875-frame
    (10 s, the utt10s workload) utterance on the FFMA path, whose conv stack is close enough to the oracle to see it."""
    u = Utt(*_synth_utt(1875, 1100), 1200)
    ref = _oracle(("phase", u.L), u)
    errs = {}
    for tc in (True, False):
        voc.set_tensor_cores(tc)
        errs["oracle_tc" if tc else "oracle_ffma"] = _maxabs(_generate(voc, [u]), ref)
    voc.set_tensor_cores(True)
    _report("10 s utterance", errs, {"oracle_tc": BAR_ORACLE[True], "oracle_ffma": BAR_PHASE})


# ---------------------------------------------------------------------------------------------------------------------
# 11,990 + 11,990 + 17 = 23,997 frames fill the first group (+5 would exceed 24,000) and 5 + 11,990 + 11,989 + 16 =
# 24,000 the second, so both group boundaries fall between two short utterances: 17 | 5 and 16 | 1.
GROUP_LENGTHS = [11990, 11990, 17, 5, 11990, 11989, 16, 1, 300]
GROUPS = [(0, 3), (3, 7), (7, 9)]


def test_grouping_matches_per_group_and_solo_calls(voc):
    voc.set_tensor_cores(True)
    assert voc.max_frames_per_call == 24000 and sum(GROUP_LENGTHS) > 24000
    utts = [Utt(*_synth_utt(L, 900 + i), 1000 + i) for i, L in enumerate(GROUP_LENGTHS)]
    wav = _split(_generate(voc, utts), utts)
    per_group = []
    for b0, b1 in GROUPS:
        assert sum(GROUP_LENGTHS[b0:b1]) <= 24000 and (b1 == len(utts) or sum(GROUP_LENGTHS[b0:b1 + 1]) > 24000)
        per_group += _split(_generate(voc, utts[b0:b1]), utts[b0:b1])
    errs = {"group": 0.0, "solo": 0.0, "oracle": 0.0}
    for i, (u, w, g) in enumerate(zip(utts, wav, per_group)):
        e, s = _maxabs(w, g), _maxabs(w, _generate(voc, [u]))
        line = f"  #{i} L={u.L:5d}: vs per-group call {e:.2e}, vs solo {s:.2e}"
        if u.L < 100:  # the utterances on either side of a group boundary
            o = _maxabs(w, _oracle(("group", i), u))
            errs["oracle"] = max(errs["oracle"], o)
            line += f", vs oracle {o:.2e}"
        print(line)
        errs["group"], errs["solo"] = max(errs["group"], e), max(errs["solo"], s)
    # a grouped call computes exactly what one call per group computes: bar 0 (as `<`, the smallest positive float)
    _report("grouping", errs, {"group": np.nextafter(0, 1), "solo": BAR_SOLO, "oracle": BAR_ORACLE[True]})


def test_batch64_grouped_equals_solo(voc):
    """The bench's batch64 workload (64 utterances, 110,119 frames): Vocoder.generate's groups against one call per
    utterance."""
    voc.set_tensor_cores(True)
    lens = [int(round(187.5 * s)) for s in synth.batch_seconds(64, seed=1234)]
    assert sum(lens) == 110119
    offs = _offs(lens)
    g = torch.Generator(device=DEV).manual_seed(64)
    n = int(offs[-1])
    mel = (-3.0 + 2.0 * torch.randn(n, 80, generator=g, device=DEV)).clamp(-6, 1.5)
    f0 = 150 + 350 * torch.rand(n, generator=g, device=DEV)
    f0[torch.rand(n, generator=g, device=DEV) < 0.2] = 0
    ini = torch.rand(64, 9, generator=g, device=DEV)
    ini[:, 0] = 0
    src = torch.randn(n * HOP, 9, generator=g, device=DEV)
    wav = voc.generate(mel, f0, offs, rand_ini=ini, src_noise=src)
    worst = 0.0
    for b in range(64):
        a, e = int(offs[b]), int(offs[b + 1])
        w = voc.generate(mel[a:e], f0[a:e], np.array([0, e - a], np.int32), rand_ini=ini[b:b + 1].contiguous(),
                         src_noise=src[a * HOP:e * HOP])
        worst = max(worst, float((wav[a * HOP:e * HOP] - w).abs().max()))
    _report("batch64 grouped vs solo", {"solo": worst}, {"solo": BAR_SOLO})


# ---------------------------------------------------------------------------------------------------------------------
TAIL = 1 << 20


def _raw_generate(v, utts, ws, ws_bytes):
    """ssb_hifigan_generate through ctypes on a caller-owned workspace."""
    from stylesinger_b200._lib import check, lib
    mel, f0, ini, src, offs = _cat(utts)
    wav = torch.empty(int(offs[-1]) * HOP, dtype=torch.float32, device=DEV)
    p = lambda t: C.c_void_p(t.data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.ssb_hifigan_generate(v._h, p(mel), p(f0), offs.ctypes.data, len(utts), p(ini), p(src), 0, p(wav), p(ws),
                                   ws_bytes, stream), "ssb_hifigan_generate")
    torch.cuda.synchronize()
    return wav


def _ws_bytes(v, utts):
    from stylesinger_b200._lib import lib
    offs = _offs([u.L for u in utts])
    n = int(lib.ssb_vocoder_workspace_bytes(v._h, offs.ctypes.data, len(utts)))
    assert n > 0
    return n


@pytest.mark.parametrize("tc", [True, False], ids=["tc", "ffma"])
def test_workspace_contract(voc, tc):
    """The caller owns the workspace and ssb_vocoder_workspace_bytes is enough: the call never reads bytes it has not
    written (a workspace of 0xFF bytes, NaN in fp32 and fp16, gives the bits a zeroed one gives), never writes past that
    size (a 1 MB sentinel tail survives), and a workspace left over from a larger call of another shape changes nothing."""
    voc.set_tensor_cores(tc)
    big, small = bench_utts(), edge_utts()
    nb, ns = _ws_bytes(voc, big), _ws_bytes(voc, small)
    print(f"workspace bytes: bench-sized call {nb}, edge batch {ns}")
    g = torch.Generator(device=DEV).manual_seed(5)
    sentinel = torch.randint(0, 256, (TAIL,), generator=g, device=DEV, dtype=torch.int32).to(torch.uint8)
    try:
        ws = torch.empty(nb + TAIL, dtype=torch.uint8, device=DEV)
        ws[nb:] = sentinel
        ws[:nb].fill_(0xFF)
        a = _raw_generate(voc, big, ws, nb)
        assert torch.equal(ws[nb:], sentinel), "the bench-sized call wrote past ssb_vocoder_workspace_bytes"
        ws[:nb].zero_()
        b = _raw_generate(voc, big, ws, nb)
        assert torch.equal(ws[nb:], sentinel)
        assert torch.isfinite(a).all() and torch.equal(a, b), "the result depends on workspace bytes the call never wrote"
        # the bench-sized call's leftovers, then the edge batch on the same workspace, vs a fresh one (zeroed, then 0xFF)
        c = _raw_generate(voc, small, ws, nb)
        del ws
        ws2 = torch.zeros(ns + TAIL, dtype=torch.uint8, device=DEV)
        ws2[ns:] = sentinel
        d = _raw_generate(voc, small, ws2, ns)
        ws2[:ns].fill_(0xFF)
        e = _raw_generate(voc, small, ws2, ns)
        assert torch.equal(ws2[ns:], sentinel), "the edge batch wrote past ssb_vocoder_workspace_bytes"
        assert torch.isfinite(c).all() and torch.equal(c, d) and torch.equal(d, e)
        print(f"workspace contract ({'tc' if tc else 'ffma'}): bit-identical on 0xFF / zeroed / reused workspaces, "
              "sentinel tails intact")
    finally:
        voc.set_tensor_cores(True)
