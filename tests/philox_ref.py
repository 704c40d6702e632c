"""NumPy restatement of the library's in-kernel noise (stylesinger_b200/csrc/philox.cuh): Philox4x32-10, the fp32
uniform and Box-Muller normal built on it, the stream plan of every draw site, and builders that lay the draws out the way
the C ABI takes injected noise.  Test-only: nothing here imports the package under test.

Key and counter placement follow `philox4`: the 64-bit counter goes in words c0/c1, the 64-bit stream id in c2/c3 and the
64-bit seed in the key k0/k1.  `uniform` is bit-exact with the kernel (the fp32 adds and multiplies are done in float32);
`normal` is Box-Muller in float64 from those fp32 uniforms, rounded to fp32, so it differs from the kernel's logf / cospif
by a few ulp only.
"""
import numpy as np

M32 = 0xFFFFFFFF
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
GROUP_SEED_STEP = 0x9E3779B97F4A7C15  # seed step between persistent mel groups (stages.cu, run_mel_diffusion)
GROUP_TILES, TILE_ROWS = 48, 128


def philox4x32_10(ctr64, stream64, seed64):
    """Philox4x32-10 of (counter, stream) under key `seed`.  ctr64 / stream64: integer arrays (broadcast together) or
    scalars; seed64: a Python int.  Returns the four uint32 output words, each shaped like the broadcast input."""
    ctr = np.asarray(ctr64, dtype=np.uint64)
    st = np.asarray(stream64, dtype=np.uint64)
    ctr, st = np.broadcast_arrays(ctr, st)
    m = np.uint64(M32)
    c0, c1 = ctr & m, ctr >> np.uint64(32)
    c2, c3 = st & m, st >> np.uint64(32)
    seed = int(seed64) & ((1 << 64) - 1)
    k0, k1 = seed & M32, seed >> 32
    for _ in range(10):
        p0 = _M0 * c0  # 32 x 32 -> 64 bits: exact in uint64
        p1 = _M1 * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & m,
                          (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & m)
        k0, k1 = (k0 + _W0) & M32, (k1 + _W1) & M32
    return tuple(w.astype(np.uint32) for w in (c0, c1, c2, c3))


def u32_to_unit_closed(x):
    """The kernel's uint32 -> fp32 grid (k + 0.5) / 2^24, k = x >> 8, in float32 arithmetic: (0, 1], the top k rounds
    to 1.  The Box-Muller inputs."""
    x = np.asarray(x, dtype=np.uint32)
    return ((x >> np.uint32(8)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 16777216.0)


def u32_to_unit(x):
    """The kernel's uniform draw: the grid with its one value 1 clamped to 1 - 2^-24, so (0, 1)."""
    return np.minimum(u32_to_unit_closed(x), np.float32(1.0 - 2.0 ** -24))


def uniform(seed, stream, ctr):
    return u32_to_unit(philox4x32_10(ctr, stream, seed)[0])


def normal_from_words(w0, w1):
    u1 = u32_to_unit_closed(w0).astype(np.float64)  # u1 = 1 gives radius 0
    u2 = u32_to_unit_closed(w1)
    two_u2 = (np.float32(2.0) * u2).astype(np.float64)  # the kernel's cospif(2.0f * u2): the product is exact in fp32
    return (np.sqrt(-2.0 * np.log(u1)) * np.cos(np.pi * two_u2)).astype(np.float32)


def normal(seed, stream, ctr):
    w = philox4x32_10(ctr, stream, seed)
    return normal_from_words(w[0], w[1])


def normal_u1(seed, stream, ctr):
    """The first uniform of each normal draw (the Box-Muller radius input), for selecting the draws near u1 = 1."""
    return u32_to_unit_closed(philox4x32_10(ctr, stream, seed)[0])


# ---- stream plan (philox.cuh) -----------------------------------------------------------------------------------------
def philox_stream(tag, sub):
    """stream = (tag << 32) | sub: the tagged range of one draw kind, sub < 2^32."""
    assert 0 <= sub < (1 << 32)
    return (tag << 32) | sub


def stream_mel_xt():
    return 1000


def stream_mel_step(t):
    return 1001 + t if t < 999 else philox_stream(2, t)


def stream_f0_xt(net):
    return 2000 + 100000 * net


def stream_f0_gauss(net, t):
    return stream_f0_xt(net) + 10 + 2 * t if t < 4000 else philox_stream(4 + net, t)


def stream_f0_unif(net, t):
    return stream_f0_xt(net) + 11 + 2 * t if t < 4000 else philox_stream(6 + net, t)


def stream_voc_ini(b):
    return 0x5151 + b if b < 8224 else philox_stream(8, b)


def stream_voc_src():
    return 0x7171


def draw_plan(T_mel, T_f0, B, sum_f=1, hop=256):
    """Every draw kind of one ssb_acoustic_forward (DDPM mel sampler, both F0 nets) plus one ssb_hifigan_generate that
    share a seed, as (name, stream, 1, counters): one entry per stream, each read at counters [0, counters)."""
    F, S = sum_f, sum_f * hop
    plan = [("mel x_T", stream_mel_xt(), 1, 80 * F)]
    plan += [(f"mel step t={t}", stream_mel_step(t), 1, 80 * F) for t in range(T_mel)]
    for n in range(2):
        plan += [(f"f0[{n}] x_T", stream_f0_xt(n), 1, F)]
        for t in range(T_f0):
            plan += [(f"f0[{n}] gauss t={t}", stream_f0_gauss(n, t), 1, F),
                     (f"f0[{n}] unif t={t}", stream_f0_unif(n, t), 1, 2 * F)]
    plan += [(f"voc rand_ini b={b}", stream_voc_ini(b), 1, 9) for b in range(B)]
    plan += [("voc source", stream_voc_src(), 1, 9 * S)]
    return plan


# ---- injected-noise layouts of the C ABI ------------------------------------------------------------------------------
def _tight(frame_offsets):
    return np.arange(int(frame_offsets[-1]), dtype=np.uint64)


def mel_noise(seed, T, frame_offsets, steps=None):
    """[(T+1), sumF, 80]: block 0 is x_T, block T-t is step t; counter ti*80 + c.  `steps`: only these step numbers t
    (other blocks left zero) - a probe reads one block."""
    ti = _tight(frame_offsets)
    ctr = ti[:, None] * np.uint64(80) + np.arange(80, dtype=np.uint64)[None, :]
    out = np.zeros((T + 1, len(ti), 80), np.float32)
    out[0] = normal(seed, stream_mel_xt(), ctr)
    for t in (range(T) if steps is None else steps):
        out[T - t] = normal(seed, stream_mel_step(t), ctr)
    return out


def mel_noise_grouped(seed, T, lens, steps=None):
    """mel_noise as the persistent mel groups draw it (ssb_model_set_persistent_groups, > 48 row tiles): greedy groups
    of consecutive utterances of <= 48 tiles of 128 rows, group g seeded seed + 0x9E3779B97F4A7C15 g (mod 2^64), rows
    indexed inside the group.  Returns (noise, number of groups)."""
    blocks, g = [], 0
    for b0, b1 in persistent_groups(lens):
        offs = np.concatenate([[0], np.cumsum(lens[b0:b1])])
        blocks.append(mel_noise((seed + GROUP_SEED_STEP * g) % (1 << 64), T, offs, steps))
        g += 1
    return np.concatenate(blocks, axis=1), g


def persistent_groups(lens):
    tiles = [(int(n) + TILE_ROWS - 1) // TILE_ROWS for n in lens]
    out, b0 = [], 0
    while b0 < len(lens):
        b1, nt = b0, 0
        while b1 < len(lens) and (b1 == b0 or nt + tiles[b1] <= GROUP_TILES):
            nt += tiles[b1]
            b1 += 1
        out.append((b0, b1))
        b0 = b1
    return out


def f0_gauss_noise(seed, net, T, frame_offsets):
    """[(T+1), sumF]: block 0 is x_T, block T-t is step t; counter ti."""
    ti = _tight(frame_offsets)
    out = np.empty((T + 1, len(ti)), np.float32)
    out[0] = normal(seed, stream_f0_xt(net), ti)
    for t in range(T):
        out[T - t] = normal(seed, stream_f0_gauss(net, t), ti)
    return out


def f0_unif_noise(seed, net, T, frame_offsets):
    """[T, sumF, 2]: block T-1-t is step t; counter 2 ti + j."""
    ti = _tight(frame_offsets)
    ctr = ti[:, None] * np.uint64(2) + np.arange(2, dtype=np.uint64)[None, :]
    out = np.empty((T, len(ti), 2), np.float32)
    for t in range(T):
        out[T - 1 - t] = uniform(seed, stream_f0_unif(net, t), ctr)
    return out


def vocoder_rand_ini(seed, B):
    """[B, 9]: column 0 is zero (the fundamental has no random phase), h >= 1 from the utterance's stream, counter h."""
    out = np.zeros((B, 9), np.float32)
    h = np.arange(1, 9, dtype=np.uint64)
    for b in range(B):
        out[b, 1:] = uniform(seed, stream_voc_ini(b), h)
    return out


def vocoder_src_noise(seed, frame_offsets, hop=256):
    """[sumF*hop, 9]: counter ti*9 + h, ti the tight sample index of the whole call."""
    n = int(frame_offsets[-1]) * hop
    ctr = np.arange(n, dtype=np.uint64)[:, None] * np.uint64(9) + np.arange(9, dtype=np.uint64)[None, :]
    return normal(seed, stream_voc_src(), ctr)


def acoustic_noise(seed, T_mel, T_f0, frame_offsets):
    """The injected-noise dict of AcousticModel.forward (numpy) that Philox mode draws for one call with `seed`."""
    return {"f0_gauss": [f0_gauss_noise(seed, n, T_f0, frame_offsets) for n in range(2)],
            "f0_unif": [f0_unif_noise(seed, n, T_f0, frame_offsets) for n in range(2)],
            "mel": mel_noise(seed, T_mel, frame_offsets)}


# ---- statistics -------------------------------------------------------------------------------------------------------
def check_stats(x, kind, streams=None):
    """Mean, variance, KS distance and lag-1 correlation of draws `x` [n_streams, n_counters] (one row per stream,
    consecutive counters along a row) against N(0,1) or U(0,1).  Every statistic must be within 5/sqrt(n) of its ideal
    value (5 sqrt(2)/sqrt(n) for a normal's relative variance, whose standard error is sqrt(2/n)).  Returns the statistics
    for printing; raises AssertionError on a miss."""
    from scipy import stats
    x = np.asarray(x, np.float64)
    if x.ndim == 1:
        x = x[None]
    flat = x.reshape(-1)
    n = flat.size
    bar = 5.0 / np.sqrt(n)
    if kind == "normal":
        mean, var, cdf = 0.0, 1.0, "norm"
    else:
        mean, var, cdf = 0.5, 1.0 / 12.0, "uniform"
    s = {"n": n, "mean": float(flat.mean() - mean), "var": float(flat.var() / var - 1.0),
         "ks": float(stats.kstest(flat, cdf).statistic)}
    z = (x - mean) / np.sqrt(var)
    s["lag1_ctr"] = float((z[:, 1:] * z[:, :-1]).mean()) if x.shape[1] > 1 else 0.0
    s["lag1_stream"] = float((z[1:] * z[:-1]).mean()) if x.shape[0] > 1 else 0.0
    for k in ("mean", "var", "ks", "lag1_ctr", "lag1_stream"):
        b = bar * (np.sqrt(2.0) if k == "var" and kind == "normal" else 1.0)
        assert abs(s[k]) < b, f"{kind}: {k} = {s[k]:.3e} outside +-{b:.3e} (n = {n})"
    return s
