"""The NumPy restatement of the in-kernel noise (tests/philox_ref.py) on its own: Random123 known answers, the uniform's
range, disjointness of the stream plan, and the statistics of the transforms.  No GPU."""
import os
import re

import numpy as np
import pytest

from tests import philox_ref as P

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "stylesinger_b200", "csrc")


def _words(ctr, key):
    """Random123 argument order: ctr = (c0, c1, c2, c3), key = (k0, k1)."""
    w = P.philox4x32_10(ctr[0] | (ctr[1] << 32), ctr[2] | (ctr[3] << 32), key[0] | (key[1] << 32))
    return [int(x) for x in w]


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox4x32_10_known_answers(ctr, key, want):
    assert _words(ctr, key) == list(want)


def test_philox_vectorised_matches_scalar_calls():
    ctr = np.array([0, 1, 2**32 - 1, 2**32, 2**63 + 5], np.uint64)
    st = np.array([7, 2**40 + 3, 0, 2**64 - 1, 12], np.uint64)
    seed = 0xDEADBEEF12345678
    vec = P.philox4x32_10(ctr, st, seed)
    for i in range(len(ctr)):
        one = P.philox4x32_10(int(ctr[i]), int(st[i]), seed)
        assert [int(w[i]) for w in vec] == [int(w) for w in one]


def test_uniform_is_strictly_inside_the_unit_interval():
    x = np.array([0, 1, 0xFF, 0x100, 0xFFFFFEFF, 0xFFFFFF00, 0xFFFFFFFE, 0xFFFFFFFF], np.uint32)
    u = P.u32_to_unit(x)
    assert u.dtype == np.float32
    print("u32_to_unit at the extremes:", [float(v) for v in u])
    assert (u > 0).all() and (u < 1).all()
    # the normals take the (0, 1] grid: at its top the Box-Muller radius is 0, a finite draw
    assert P.u32_to_unit_closed(np.uint32(0xFFFFFFFF)) == 1.0
    z = P.normal_from_words(np.full(4, 0xFFFFFFFF, np.uint32), np.array([0, 1 << 30, 1 << 31, 3 << 30], np.uint32))
    assert np.isfinite(z).all() and (z == 0).all()


def test_uniform_mapping_is_the_half_cell_grid_clamped_below_one():
    """u = (k + 0.5) / 2^24 for k = x >> 8, rounded to fp32 (above 2^23 the sum k + 0.5 is not representable), monotone,
    and the one value that rounds up to 1 clamped to 1 - 2^-24."""
    x = np.random.default_rng(0).integers(0, 2**32, 1 << 16, dtype=np.uint64).astype(np.uint32)
    x = np.sort(np.concatenate([x, [0, 0xFFFFFE00, 0xFFFFFEFF, 0xFFFFFF00, 0xFFFFFFFF]]).astype(np.uint32))
    u = P.u32_to_unit(x).astype(np.float64)
    k = (x >> np.uint32(8)).astype(np.float64)
    assert (np.diff(u) >= 0).all()
    assert (np.abs(u - (k + 0.5) / 2.0**24) <= 2.0**-25).all()
    assert u.max() == 1.0 - 2.0**-24 and u.min() == 2.0**-25


def test_stream_plan_keeps_the_legacy_ids_where_they_cannot_collide():
    """A seed keeps producing what earlier releases drew, except for the draws whose legacy stream ran into another kind's
    (mel steps t >= 999, vocoder utterances b >= 8224), which move to their tagged ranges."""
    assert P.stream_mel_xt() == 1000
    assert [P.stream_mel_step(t) for t in (0, 99, 998)] == [1001, 1100, 1999]
    assert P.stream_mel_step(999) == (2 << 32) | 999
    assert [P.stream_f0_xt(n) for n in (0, 1)] == [2000, 102000]
    assert (P.stream_f0_gauss(1, 99), P.stream_f0_unif(1, 99)) == (102208, 102209)
    assert P.stream_f0_gauss(0, 3999) == 2010 + 2 * 3999 and P.stream_f0_unif(0, 4000) == (6 << 32) | 4000
    assert P.stream_voc_ini(8223) == 0x7170 and P.stream_voc_ini(8224) == (8 << 32) | 8224 and P.stream_voc_src() == 0x7171


@pytest.mark.parametrize("T_mel", [1, 100, 999, 1000, 1009, 4000])
@pytest.mark.parametrize("T_f0", [1, 100, 999, 1000, 1009, 4000, 4001])
def test_stream_plan_is_disjoint(T_mel, T_f0):
    """No two draw kinds of one acoustic forward plus one vocoder call sharing a seed ever read the same (stream, counter):
    the kinds are compared stream by stream, for batches of up to 2^16 utterances."""
    B = 1 << 16
    plan = P.draw_plan(T_mel, T_f0, B)
    lo = np.array([p[1] for p in plan], np.uint64)
    hi = lo + np.array([p[2] for p in plan], np.uint64)
    order = np.argsort(lo, kind="stable")
    lo, hi = lo[order], hi[order]
    clash = np.nonzero(hi[:-1] > lo[1:])[0]
    msg = [f"{plan[order[i]][0]} [{int(lo[i])}, {int(hi[i])}) meets {plan[order[i + 1]][0]} at stream {int(lo[i + 1])}"
           for i in clash[:3]]
    assert clash.size == 0, "; ".join(msg)


def test_layouts_follow_the_abi_block_order():
    offs = np.array([0, 3, 8], np.int32)
    T, seed = 3, 11
    mel = P.mel_noise(seed, T, offs)
    assert mel.shape == (T + 1, 8, 80)
    ti, c = 6, 17
    assert mel[0, ti, c] == P.normal(seed, P.stream_mel_xt(), ti * 80 + c)
    assert mel[T - 1, ti, c] == P.normal(seed, P.stream_mel_step(1), ti * 80 + c)
    g = P.f0_gauss_noise(seed, 1, T, offs)
    assert g[0, ti] == P.normal(seed, P.stream_f0_xt(1), ti) and g[T, ti] == P.normal(seed, P.stream_f0_gauss(1, 0), ti)
    u = P.f0_unif_noise(seed, 0, T, offs)
    assert u.shape == (T, 8, 2)
    assert u[T - 1, ti, 1] == P.uniform(seed, P.stream_f0_unif(0, 0), 2 * ti + 1)  # step 0 is the LAST block
    assert u[0, ti, 0] == P.uniform(seed, P.stream_f0_unif(0, T - 1), 2 * ti)
    ini = P.vocoder_rand_ini(seed, 2)
    assert (ini[:, 0] == 0).all() and ini[1, 4] == P.uniform(seed, P.stream_voc_ini(1), 4)
    src = P.vocoder_src_noise(seed, offs, hop=4)
    assert src.shape == (32, 9) and src[21, 5] == P.normal(seed, P.stream_voc_src(), 21 * 9 + 5)


def test_persistent_group_split_and_seeds():
    lens = [1000 + 37 * i for i in range(12)]
    groups = P.persistent_groups(lens)
    assert groups[0][0] == 0 and groups[-1][1] == len(lens) and len(groups) > 1
    for b0, b1 in groups:
        tiles = sum((n + 127) // 128 for n in lens[b0:b1])
        assert tiles <= 48 or b1 == b0 + 1
    noise, ng = P.mel_noise_grouped(5, 2, lens, steps=[1])
    b0, b1 = groups[1]
    a = sum(lens[:b0])
    seed1 = (5 + 0x9E3779B97F4A7C15) % (1 << 64)
    assert noise[1, a + 3, 7] == P.normal(seed1, P.stream_mel_step(1), 3 * 80 + 7)  # group-local row 3
    assert ng == len(groups)


def test_transform_statistics():
    """A few million restated draws: N(0,1) and U(0,1) moments, KS distance and lag-1 correlation along consecutive
    counters and across adjacent streams, all within 5 standard errors (fixed seeds: deterministic)."""
    ctr = np.arange(1 << 18, dtype=np.uint64)
    st = np.arange(8, dtype=np.uint64)[:, None]
    for seed in (0, 0x1234567890ABCDEF):
        z = P.normal(seed, P.stream_mel_step(0) + st, ctr[None])
        u = P.uniform(seed, P.stream_f0_unif(0, 0) + st, ctr[None])
        print("normal", P.check_stats(z, "normal"))
        print("uniform", P.check_stats(u, "uniform"))


def test_check_stats_rejects_a_correlated_stream():
    z = P.normal(3, P.stream_mel_xt(), np.arange(1 << 16, dtype=np.uint64))
    with pytest.raises(AssertionError):
        P.check_stats(np.stack([z, z]), "normal")  # two identical "streams"
    with pytest.raises(AssertionError):
        P.check_stats(z * np.float32(1.02), "normal")


def _calls(txt, name):
    """Argument lists (split at top-level commas) of every call of `name` in `txt`."""
    out = []
    for m in re.finditer(r"(?<![\w.])" + name + r"\s*\(", txt):
        i, depth, args, cur = m.end(), 1, [], ""
        while depth:
            ch = txt[i]
            depth += ch == "("
            depth -= ch == ")"
            if depth and ch == "," and depth == 1:
                args.append(cur.strip())
                cur = ""
            elif depth:
                cur += ch
            i += 1
        out.append(args + [cur.strip()])
    return out


def test_stream_ids_are_formed_only_in_philox_cuh():
    """Every Philox stream id comes from a stream_* function of philox.cuh: outside that header a stream argument or
    field is only ever such a call or a variable passing one through (no literal, no stream arithmetic)."""
    plan = r"stream_(?:mel_xt|mel_step|f0_xt|f0_gauss|f0_unif|voc_ini|voc_src)\([^()]*\)"
    passthrough = r"(?:[A-Za-z_]\w*\.)?(?:stream_id|stream2|gauss_stream|unif_stream|sid)"
    ok = re.compile(rf"^(?:{plan}|{passthrough})$")
    bad, seen = [], 0
    # the stream position of each host-side wrapper (ops.cuh) and of the device draws
    wrappers = {"mel_q_sample": 12, "mel_p_sample": 9, "f0_init": 6, "philox_normal": 1, "philox_uniform": 1}
    for f in sorted(os.listdir(CSRC)):
        if f == "philox.cuh" or not f.endswith((".cu", ".cuh")):
            continue
        txt = re.sub(r"//[^\n]*", "", open(os.path.join(CSRC, f)).read())
        for name, pos in wrappers.items():
            for args in _calls(txt, name):
                if any(a.startswith(("Ctx", "uint64_t", "const ")) for a in args):
                    continue  # a declaration
                seen += 1
                if len(args) <= pos or not ok.match(args[pos]):
                    bad.append(f"{f}: {name}(... {args[pos] if len(args) > pos else args} ...)")
        for m in re.finditer(r"\b(?:stream_id|stream2|gauss_stream|unif_stream)\s*=\s*(\w+\([^()]*\)|[^;,]+)", txt):
            v = m.group(1).strip()
            if v != "0" and not re.match(rf"^{plan}$", v):
                bad.append(f"{f}: stream set to {v!r}")
            seen += 1
    assert seen >= 15
    assert not bad, "\n".join(bad)
