"""The diffusion denoisers and their reverse steps against the float64 restatement (tests/denoiser_oracle.py), on every
kernel path, at bench size and at tile edges.

(a) Single evaluations (ssb_denoiser_eval) of the mel DiffNet and the two F0 DDiffNets at t in {0, 50, 99} of T = 100,
on the tensor-core path and on the fp32 FFMA path, at three sizes: small (< 8 row tiles), mid (71 row tiles: the mel
layers on the CTA-pair kernels tc2r<64,GATE> / tc2<64,RES_SKIP>, the F0 layers, N = 384, on tc<64,.>) and the bench's
batch64 utterances (890 row tiles, every layer GEMM on the CTA-pair kernels).  The lengths include 1, 2, 3, 8, 9, 16,
17, 127, 128 and 129 frames: the row tile is 128 frames, the dilated taps reach 8 rows and the guard band between
utterances is 16 rows.  Every call asserts the tensor-core GEMM variants it launched (a restatement of conv_gemm_tc's
dispatch), so that a threshold change cannot move a test off its path.  Errors on the 8 rows at each utterance end are
reported apart from the interior; an edge error above 4x the interior error fails whatever the bar, since that is what
a guard-row or neighbour-tile write looks like.  Small and mid utterances are also run as their own B = 1 calls: FFMA
must be bit-identical, tensor cores within the bar.

(b) Short reverse chains, where the sampler update itself is visible: the mel DDPM sampler at K_step in {1, 2, 4} of
T = 100 (steps with injected noise and the noiseless t = 0) on the persistent single launch, per-launch tensor cores and
FFMA; both F0 samplers (f0_T = 4) per launch and on FFMA; the persistent two-net F0 kernel through ssb_acoustic_forward.
A UV decision may differ from the float64 chain only where the float64 Gumbel margin at some step is below 1e-4; z is
compared on frames out of reach of such a frame.  Each chain prints the fraction of x0 predictions the clip changed and
asserts that both branches of the clip are taken: about 6 % of the mel predictions are clipped, while the F0 band is
+-3 semitones around the note, so the early F0 steps clip most predictions and the last about half.

Errors are max |a - b| / max(1, |b|).  Each bar is at most 4x the largest error measured on an H100 SXM (80 GB), with
the measured value beside it; each test prints what it measured.
"""
import time

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from tests import denoiser_oracle as DO
from tests.common import acoustic_engine, hp_for
from tests.gpu_checks import (Err, check_variants, cond_gemm, count, frame_offsets, launched, net_dims, ntiles,
                              rel, split, step_gemms)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T = 100
STEPS = (0, 50, 99)
F0_T = 4
RF = 33  # rows one DDiffNet evaluation reaches on each side: the dilations 1, 2, 4, 8, 1, 2, 4, 8, 1, 2 summed
MARGIN = 1e-4

# measured on an H100 80GB HBM3 (SXM, 700 W power limit); the largest error over the three nets, t and sizes is beside
# each bar.  0 means bit-identical.
BARS = {
    "eval": {"ffma": 5e-6,                       # 1.4e-6 (mel, bench)
             "tc": 2.2e-5},                      # 6.0e-6 (mel, bench)
    "solo": {"ffma": 0.0,
             "tc": 4.5e-6},                      # 1.2e-6 (mel, mid: the batch takes the CTA-pair kernels, B = 1 not)
    "mel_chain": {"ffma": 4.5e-6,                # 1.1e-6 (mel_out, K = 4)
                  "tc": 7.5e-6,                  # 1.9e-6
                  "persistent": 6e-6},           # 1.6e-6
    "f0_chain": {"ffma": 8e-7,                   # 2.0e-7
                 "tc": 3.5e-6,                   # 8.9e-7
                 "persistent": 4.5e-7},          # 1.2e-7 (pitch_pred)
}

EDGE = [1, 2, 3, 8, 9, 16, 17, 127, 128, 129]
SMALL = [129, 1, 2, 8, 17, 127]                                                  # 7 row tiles
MID = [129, 1, 2000, 2, 3, 8, 1500, 9, 16, 17, 3000, 127, 128, 900]             # 71 row tiles
RAGGED = [129, 1, 2, 3, 8, 9, 16, 17, 127, 128, 700]                             # 17 row tiles
TILES48 = [EDGE[i % 9] for i in range(48)]                                       # 48 utterances, one row tile each


def expected_eval(which, lens):
    return count(cond_gemm(which) + step_gemms(which), ntiles(lens))


# ---------------------------------------------------------------------------------------------------------------------
# inputs: synthetic utterances through the forward (mel diffusion skipped) for diff_cond and the coarse mel
_B = {}


def _utts(lens, base):
    return [synth.make_utterance(n / 187.5, utt_idx=base + i, ref_frames=64, frames=n, phones=max(1, min(n // 6, 60)))
            for i, n in enumerate(lens)]


def batch(name):
    """{utts, lens, offs, cond [sumF,256], coarse [sumF,80], midi [sumF]} (device tensors), memoised."""
    if name not in _B:
        from stylesinger_b200.engine import pack_batch
        if name in ("bench", "bench6"):
            utts = [synth.make_utterance(float(s), utt_idx=i) for i, s in enumerate(synth.batch_seconds(64, seed=1234))]
            if name == "bench6":  # the shortest, the longest and four others
                lens = [len(u["mel2ph"]) for u in utts]
                pick = sorted({int(np.argmin(lens)), int(np.argmax(lens)), 5, 21, 40, 63})
                utts = [utts[i] for i in pick]
        else:
            lens = {"small": SMALL, "mid": MID, "ragged": RAGGED, "tiles48": TILES48}[name]
            utts = _utts(lens, 700 + 100 * len(_B))
        pb = pack_batch(utts).to(DEV)
        m = acoustic_engine(T, F0_T)
        out = m.forward(pb, seed=1, skip_mel_diffusion=True, want=("diff_cond", "coarse_mel"))
        lens = [len(u["mel2ph"]) for u in utts]
        midi = torch.cat([u["note"][u["mel2ph"] - 1] * (u["mel2ph"] > 0) for u in utts]).float()
        _B[name] = dict(utts=utts, lens=lens, offs=frame_offsets(lens), pb=pb, cond=out["diff_cond"].clone(),
                        coarse=out["coarse_mel"].clone(), midi=midi)
        if name == "bench":
            assert int(_B[name]["offs"][-1]) == 110119 and ntiles(lens) == 890
    return _B[name]


def eval_inputs(which, t, b):
    """mel: x_t = sqrt(ac_t) norm_spec(coarse) + sqrt(1 - ac_t) eps; F0: z in [-1, 1] and a random uv."""
    g = torch.Generator().manual_seed(1000 * which + t)
    n = int(b["offs"][-1])
    if which == 0:
        s = O._gauss_tables(T, hp_for(T)["max_beta"])
        smin, smax = DO.spec_bounds(hp_for(T))
        x0 = (b["coarse"].cpu().double() - smin) / (smax - smin) * 2 - 1
        x = float(s["sqrt_alphas_cumprod"][t]) * x0 + float(s["sqrt_one_minus_alphas_cumprod"][t]) * torch.randn(
            n, 80, generator=g, dtype=torch.float64)
        return x.float().to(DEV), None
    z = 2 * torch.rand(n, generator=g) - 1
    uv = (torch.rand(n, generator=g) < 0.3).int()
    return z.to(DEV), uv.to(DEV)


_OR = {}


def _f64_eval(which, t, name, i, x, uv, cond):
    key = (which, t, name, i)
    if key not in _OR:
        hp = hp_for(T)
        c = cond.t()[None]
        if which == 0:
            _OR[key] = DO.diffnet64(x.t()[None, None], t, c, hp)[0, 0].t()
        else:
            _OR[key] = DO.ddiffnet64(x[None, None], uv.long()[None], t, c, hp, DO.F0_PREFIX[which - 1])[0].t()
    return _OR[key]


def _compared(name, which, t, lens):
    """Utterances compared against float64: all of them, except at bench size, where every utterance is compared at one
    t per net and the shortest, the longest and every eighth at the other two."""
    if name != "bench" or t == STEPS[which]:
        return range(len(lens))
    return sorted({int(np.argmin(lens)), int(np.argmax(lens))} | set(range(0, len(lens), 8)))


# ---------------------------------------------------------------------------------------------------------------------
# (a) single evaluations
@pytest.mark.parametrize("size", ["small", "mid", "bench"])
@pytest.mark.parametrize("which", [0, 1, 2], ids=["mel", "f0_agnostic", "f0_specific"])
def test_denoiser_eval_matches_float64(which, size):
    b = batch(size)  # (its forward runs the F0 samplers at f0_T = F0_T)
    m = acoustic_engine(T)
    lens, offs = b["lens"], b["offs"]
    want = expected_eval(which, lens)
    if size == "mid":
        assert want[f"tc{'2r<64' if which == 0 else '<64'},GATE>"] == net_dims(which)[1], want
    if size == "bench":
        assert want["tc2r<64,GATE>"] == net_dims(which)[1] and want["tc2<64,RES_SKIP>"] == net_dims(which)[1], want
    t64 = 0.0
    try:
        for t in STEPS:
            x, uv = eval_inputs(which, t, b)
            xs, uvs, cs = split(x, offs), (split(uv, offs) if uv is not None else None), split(b["cond"], offs)
            outs = {}
            for path in ("tc", "ffma"):
                m.set_tensor_cores(path == "tc")
                outs[path], got, _ = launched(lambda: m.denoiser_eval(which, x, uv, t, b["cond"], offs).clone())
                check_variants(f"eval net {which} {size} t={t} {path}", got, want if path == "tc" else {})
            for path in ("tc", "ffma"):
                err, solo = Err(), 0.0
                ys = split(outs[path], offs)
                t0 = time.time()
                for i in _compared(size, which, t, lens):
                    err.add(i, ys[i], _f64_eval(which, t, size, i, xs[i], uvs[i] if uvs else None, cs[i]))
                t64 += time.time() - t0
                if size != "bench":
                    m.set_tensor_cores(path == "tc")
                    for i in range(len(lens)):
                        y1 = m.denoiser_eval(which, xs[i].to(DEV).contiguous(),
                                             uvs[i].to(DEV).contiguous() if uvs else None, t, cs[i].to(DEV).contiguous(),
                                             frame_offsets([lens[i]]))
                        e = float(rel(y1, ys[i]).max())
                        solo = max(solo, e)
                        if path == "ffma":
                            assert torch.equal(y1.cpu(), ys[i]), (size, which, t, i, e)
                    print(f"eval net {which} {size} t={t} {path}: solo B=1 calls {solo:.3e} (bar {BARS['solo'][path]:.1e})")
                    assert solo <= BARS["solo"][path]
                err.report(f"eval net {which} {size} t={t} {path} ({len(lens)} utterances, {ntiles(lens)} row tiles)",
                           BARS["eval"][path])
    finally:
        m.set_tensor_cores(True)
    print(f"eval net {which} {size}: float64 reference took {t64:.1f} s")


# ---------------------------------------------------------------------------------------------------------------------
# (b) reverse chains
def _mel_noise(K, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(K + 1, n, 80, generator=g)


_CH = {}


def _chain_coarse(name, n):
    """A coarse mel mostly inside [spec_min, spec_max] (the random model's own coarse_mel is mostly outside it, so that
    nearly every x0 prediction would be clipped): both branches of the clip are taken."""
    g = torch.Generator().manual_seed(len(name) * 7919 + n)
    return (-3 + 1.5 * torch.randn(n, 80, generator=g)).clamp(-6, 1).to(DEV)


def _mel64(name, K, b, coarse, noise):
    key = ("mel", name, K)
    if key not in _CH:
        hp = dict(hp_for(T), K_step=K)
        cs, co = split(b["cond"], b["offs"]), split(coarse, b["offs"])
        a = b["offs"]
        _CH[key] = [DO.mel_chain64(cs[i], co[i], hp, K, noise[:, int(a[i]):int(a[i + 1])]) for i in range(len(cs))]
    return _CH[key]


@pytest.mark.parametrize("K", [1, 2, 4])
def test_mel_sampler_chain_matches_float64(K):
    m = acoustic_engine(T, F0_T)
    m.set_mel_k_step(K)
    try:
        for name in ("one_tile", "ragged", "tiles48", "bench6"):
            b = batch(name) if name != "one_tile" else _one_tile()
            lens, offs = b["lens"], b["offs"]
            nt = ntiles(lens)
            noise = _mel_noise(K, int(offs[-1]), 50 + K)
            coarse = _chain_coarse(name, int(offs[-1]))
            t0 = time.time()
            ref = _mel64(name, K, b, coarse, noise)
            t64 = time.time() - t0
            clip = np.mean([np.mean(r["clip"]) for r in ref])
            print(f"mel chain {name} K={K}: float64 took {t64:.1f} s, x0 clipped in {clip:.3f} of the elements "
                  f"(per step, first utterance: {[round(c, 3) for c in ref[0]['clip']]})")
            assert 0 < clip < 0.5
            paths = (["persistent"] if nt <= 48 else []) + ["tc", "ffma"]
            for path in paths:
                m.set_tensor_cores(path != "ffma")
                m.set_persistent(path == "persistent")
                mel, got, launches = launched(lambda: m.mel_diffusion(b["cond"], coarse, offs, noise.to(DEV)).clone())
                if path == "persistent":
                    print(f"mel chain {name} K={K} persistent: {launches} launches")
                    assert launches < 16
                    want = count(cond_gemm(0), nt)
                elif path == "tc":
                    want = count(cond_gemm(0) + step_gemms(0) * K, nt)
                else:
                    want = {}
                check_variants(f"mel chain {name} K={K} {path}", got, want)
                err = Err()
                for i, y in enumerate(split(mel, offs)):
                    err.add(i, y, ref[i]["mel"])
                err.report(f"mel chain {name} K={K} {path} ({len(lens)} utterances, {nt} row tiles)",
                           BARS["mel_chain"][path])
    finally:
        m.set_tensor_cores(True)
        m.set_persistent(True)
        m.set_mel_k_step(0)


def _one_tile():
    if "one_tile" not in _B:
        b = batch("small")
        i = b["lens"].index(127)
        a, e = int(b["offs"][i]), int(b["offs"][i + 1])
        _B["one_tile"] = dict(lens=[127], offs=frame_offsets([127]), cond=b["cond"][a:e].contiguous(),
                              coarse=b["coarse"][a:e].contiguous(), midi=b["midi"][a:e])
    return _B["one_tile"]


def _f0_noise(n, seed):
    g = torch.Generator().manual_seed(seed)
    gauss = torch.randn(F0_T + 1, n, generator=g)
    unif = torch.rand(F0_T, n, 2, generator=g)
    return gauss, unif


def _uv_z_check(tag, lens, offs, uv_gpu, z_gpu, chains, bar):
    """UV decisions may differ only where the float64 margin at some step is < MARGIN (counted and printed); z is
    compared on frames out of reach of every such frame.  chains[i] is a list of f0_chain64 results whose final
    (z, uv) are combined by combine(zs, uvs) into what the GPU returns."""
    err, flips, near_total = Err(), [], 0
    for i, (n, (zref, uvref, margin)) in enumerate(zip(lens, chains)):
        a = int(offs[i])
        near = margin < MARGIN
        near_total += int(near.sum())
        zone = near.clone()
        for j in torch.nonzero(near)[:, 0].tolist():
            zone[max(0, j - RF * F0_T): j + RF * F0_T + 1] = True
        ug = uv_gpu[a:a + n]
        d = ug != uvref
        assert not (d & ~zone).any(), (tag, i, torch.nonzero(d & ~zone)[:, 0].tolist())
        for j in torch.nonzero(d)[:, 0].tolist():
            flips.append((i, j, float(margin[j])))
        keep = ~zone
        if keep.any():
            err.add(i, z_gpu[a:a + n][keep][:, None], zref[keep][:, None])
    print(f"{tag}: {near_total} frames with a float64 margin < {MARGIN}, {len(flips)} UV differences "
          f"(utterance, frame, margin) {flips}")
    err.report(tag, bar)


@pytest.mark.parametrize("which", [0, 1], ids=["agnostic", "specific"])
def test_f0_sampler_chain_matches_float64(which):
    m = acoustic_engine(T, F0_T)
    hp = hp_for(T, F0_T)
    try:
        for name in ("small", "mid", "bench6"):
            b = batch(name)
            lens, offs = b["lens"], b["offs"]
            n = int(offs[-1])
            lo, hi = (v.reshape(n) for v in O.midi_clip_band(b["midi"][None, None]))
            gauss, unif = _f0_noise(n, 60 + which)
            t0 = time.time()
            chains, clip = [], []
            for i, c in enumerate(split(b["cond"], offs)):
                a, e = int(offs[i]), int(offs[i + 1])
                r = DO.f0_chain64(c.t(), lo[a:e], hi[a:e], hp, DO.F0_PREFIX[which], gauss[:, a:e], unif[:, a:e])
                chains.append((r["z"][-1], r["uv"][-1], torch.stack(r["margin"]).min(0).values))
                clip.append(r["clip"])
            clip = np.array(clip)
            print(f"f0 chain net {which} {name}: float64 took {time.time() - t0:.1f} s, x0 clipped per step "
                  f"{np.round(clip.mean(0), 3).tolist()}")
            assert 0 < clip.mean() < 1
            for path in ("tc", "ffma"):
                m.set_tensor_cores(path == "tc")
                (z, uv), got, _ = launched(lambda: m.f0_diffusion(which, b["cond"], lo.to(DEV).contiguous(),
                                                                   hi.to(DEV).contiguous(), offs, gauss.to(DEV),
                                                                   unif.to(DEV).contiguous()))
                nt = ntiles(lens)
                check_variants(f"f0 chain net {which} {name} {path}", got,
                                count(cond_gemm(1) + step_gemms(1) * F0_T, nt) if path == "tc" else {})
                _uv_z_check(f"f0 chain net {which} {name} {path} ({len(lens)} utterances, {nt} row tiles)", lens, offs,
                            uv.cpu().long(), z.cpu().double(), chains, BARS["f0_chain"][path])
    finally:
        m.set_tensor_cores(True)


def test_f0_pair_persistent_through_forward_matches_float64():
    """Both F0 samplers in one persistent launch (ssb_acoustic_forward, <= 48 row tiles): pitch_pred against the float64
    chains on the conditioners O.stylesinger_forward composes, rebuilt from the forward's own encoder_out, spk / emo
    projections and style."""
    m = acoustic_engine(T, F0_T)
    hp = hp_for(T, F0_T)
    b = batch("ragged")
    lens, offs, pb = b["lens"], b["offs"], b["pb"]
    n = int(offs[-1])
    gauss, unif = zip(*(_f0_noise(n, 70 + k) for k in range(2)))
    noise = {"f0_gauss": [g.to(DEV).contiguous() for g in gauss], "f0_unif": [u.to(DEV).contiguous() for u in unif]}
    m.set_persistent(True)
    m.set_tensor_cores(True)
    out, got, _ = launched(lambda: m.forward(pb, noise=noise, skip_mel_diffusion=True, want=(
        "pitch_pred", "encoder_out", "spk_proj", "emo_proj", "style")))
    print(f"f0 pair persistent: tensor-core GEMM variants launched {got}")
    assert not any("GATE" in k or "RES_SKIP" in k for k in got), got  # the layer GEMMs ran inside the persistent kernel
    enc = split(out["encoder_out"], pb.ph_offsets)
    sty = split(out["style"], offs)
    spk, emo = out["spk_proj"].cpu(), out["emo_proj"].cpu()
    lo, hi = (v.reshape(n) for v in O.midi_clip_band(b["midi"][None, None]))
    f0c, uvc, clip = [], [], []
    for i, u in enumerate(b["utts"]):
        a, e = int(offs[i]), int(offs[i + 1])
        m2p = u["mel2ph"]
        tgt = (m2p > 0).double()[:, None]
        dec = enc[i].double()[(m2p - 1).clamp(min=0)] * tgt
        conds = (dec, (dec + spk[i].double() + emo[i].double() + sty[i].double()) * tgt)
        rs = [DO.f0_chain64(conds[k].t(), lo[a:e], hi[a:e], hp, DO.F0_PREFIX[k], gauss[k][:, a:e], unif[k][:, a:e])
              for k in range(2)]
        clip.append(np.mean([r["clip"] for r in rs]))
        unvoiced = b["midi"][a:e] == 0
        f0s = [(r["z"][-1] + 1) / 2 * 4 + 6 for r in rs]
        uvs = [torch.where(unvoiced, torch.ones_like(r["uv"][-1]), r["uv"][-1]) for r in rs]
        margin = torch.minimum(*(torch.stack(r["margin"]).min(0).values for r in rs))
        f0c.append(((f0s[0] + f0s[1]) / 2, uvs[0] + uvs[1], margin))
    print(f"f0 pair persistent: x0 clipped in {np.mean(clip):.3f} of the predictions")
    pp = out["pitch_pred"].cpu().double()
    # pitch_pred[:, 1] is the mean of the two UV decisions: compare their sum (0, 1, 2)
    _uv_z_check(f"f0 pair persistent ({len(lens)} utterances, {ntiles(lens)} row tiles)", lens, offs,
                (2 * pp[:, 1]).round().long(), pp[:, 0], f0c, BARS["f0_chain"]["persistent"])
