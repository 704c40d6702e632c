"""Pin the float64 denoiser restatement (tests/denoiser_oracle.py) on the CPU: the three denoisers against the reference's
own single evaluations, and the two reverse-step chains against the fp32 oracle on the same draws."""
import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from tests import denoiser_oracle as DO
from tests.common import acoustic_sd, golden, hp_for, utt_from_meta

TOL = 2e-5  # the fp32 oracle's bar against the reference (tests/test_oracle_golden.py)
MARGIN = 1e-4  # a UV decision closer than this may round either way in fp32


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


@pytest.mark.parametrize("name", ["ref_small_T4", "ref_f64_T25", "ref_f32_T100"])
def test_float64_denoisers_match_reference_fixtures(name):
    """dn_out = DiffNet(dn_spec, T-1, dn_cond); dd_out / dd_out_inp = the two DDiffNets at t = 1 / 0 (tools/make_golden.py)."""
    g, meta = golden(name)
    hp = hp_for(meta["T"])
    cond = torch.from_numpy(g["dn_cond"])[None]
    f0, uv = torch.from_numpy(g["dd_f0"])[None, None], torch.from_numpy(g["dd_uv"])[None]
    e = {"dn_out": _maxabs(DO.diffnet64(torch.from_numpy(g["dn_spec"])[None, None], meta["T"] - 1, cond, hp)[0, 0],
                           g["dn_out"]),
         "dd_out": _maxabs(DO.ddiffnet64(f0, uv, 1, cond, hp, DO.F0_PREFIX[0])[0], g["dd_out"]),
         "dd_out_inp": _maxabs(DO.ddiffnet64(f0, uv, 0, cond, hp, DO.F0_PREFIX[1])[0], g["dd_out_inp"])}
    print(name, {k: f"{v:.2e}" for k, v in e.items()})
    assert max(e.values()) < TOL, e


def _inputs(Fr, seed):
    u = utt_from_meta({"frames": Fr, "utt_idx": 300 + seed, "ref_frames": 32, "phones": 6})
    gen = torch.Generator().manual_seed(seed)
    cond = 0.5 * torch.randn(Fr, 256, generator=gen)
    coarse = (-3 + 1.5 * torch.randn(Fr, 80, generator=gen)).clamp(-6, 1.0)
    midi = u["note"][u["mel2ph"] - 1].float()
    return cond, coarse, midi


@pytest.mark.parametrize("T,K", [(100, 4), (4, 4), (100, 1)])
def test_mel_chain64_matches_fp32_oracle(T, K):
    hp = hp_for(T)
    hp["K_step"] = K
    cond, coarse, _ = _inputs(70, T + K)
    ns = O.NoiseSource(7 + K)
    ns.record = []
    with torch.no_grad():
        mel32, steps = O.mel_diffusion_sample(cond[None], coarse[None], acoustic_sd(), hp, ns, return_steps=True)
    noise = torch.stack([n[0, 0].t() for n in ns.record])
    assert noise.shape == (K + 1, 70, 80)
    r = DO.mel_chain64(cond, coarse, hp, K, noise)
    e = [_maxabs(r["x"][k + 1], steps[k][0, 0].t()) for k in range(K)]
    e_mel = _maxabs(r["mel"], mel32[0])
    print(f"mel chain T={T} K={K}: x_t err per step {[f'{v:.1e}' for v in e]}, mel {e_mel:.1e}, clip {r['clip']}")
    assert max(e) < TOL and e_mel < 4 * TOL
    assert 0 < max(r["clip"]) and min(r["clip"]) < 0.5


@pytest.mark.parametrize("which,T", [(0, 4), (1, 4), (1, 25)])
def test_f0_chain64_matches_fp32_oracle(which, T):
    hp = hp_for(4, T)
    Fr = 90
    cond, _, midi = _inputs(Fr, 40 + T + which)
    lo, hi = O.midi_clip_band(midi[None, None])
    ns = O.NoiseSource(100 + T + which)
    ns.record = []
    with torch.no_grad():
        out32 = O.f0_diffusion_sample(cond.t()[None], (lo, hi), acoustic_sd(), hp, DO.F0_PREFIX[which], ns)[0]
    rec = ns.record[1:]  # record[0] is the UV initialisation draw, never read
    gauss = torch.stack([rec[0].reshape(Fr)] + [rec[1 + 2 * k].reshape(Fr) for k in range(T)])
    unif = torch.stack([rec[2 + 2 * k][0].t() for k in range(T)])
    r = DO.f0_chain64(cond.t(), lo.reshape(Fr), hi.reshape(Fr), hp, DO.F0_PREFIX[which], gauss, unif)
    near = torch.stack(r["margin"]).min(0).values < MARGIN
    uv32 = out32[:, 1].long()
    diff = uv32 != r["uv"][-1]
    assert not (diff & ~near).any(), torch.nonzero(diff & ~near)
    keep = ~near
    e_z = _maxabs(out32[keep, 0], r["z"][-1][keep])
    print(f"f0 chain {DO.F0_PREFIX[which]} T={T}: z err {e_z:.1e}, {int(near.sum())} frames with a margin < {MARGIN}, "
          f"{int(diff.sum())} UV differences, clip {[round(c, 3) for c in r['clip']]}, "
          f"min margin {float(torch.stack(r['margin']).min()):.1e}")
    assert e_z < TOL
    assert 0 < max(r["clip"]) and min(r["clip"]) < 1
    assert 0 < int(r["uv"][-1].sum()) < Fr  # both UV classes are reached
