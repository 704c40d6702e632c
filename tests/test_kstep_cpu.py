"""Shallow diffusion (hparams['K_step'] < timesteps), CPU side: the oracle's K-step samplers against the
unmodified reference's fixture (tests/golden/ref_kstep.npz, tools/make_golden.py kstep), K_step == timesteps as the
full-schedule run, and the hparams rules.  Bars: tests/test_oracle_golden.py's (TOL per operator, 5e-5 for the T=25
sampler, TOL * max(1, |mel|) for PLMS)."""
import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200.hparams import resolve
from tests.common import acoustic_sd, golden, kstep_hp, utt_from_meta

TOL = 2e-5


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def _log(ns):
    return [[k, list(sh)] for k, sh in ns.log]


def test_full_forward_matches_reference():
    """(a) a B = 1 forward at timesteps 25, K_step 11, mel2ph given."""
    g, meta = golden("ref_kstep")
    hp = kstep_hp(meta["T_fwd"], meta["K_fwd"])
    u = utt_from_meta(meta)
    ns = O.NoiseSource(meta["seed"])
    with torch.no_grad():
        r = O.stylesinger_forward(acoustic_sd(), hp, u["txt_tokens"][None], u["note"][None], u["note_dur"][None],
                                  u["note_type"][None], u["spk_embed"][None], u["emo_embed"][None], u["ref_mels"][None],
                                  u["ref_f0"], ns, mel2ph=u["mel2ph"][None])
    assert _log(ns) == meta["noise_log"]
    # the mel sampler's draws: q_sample + K_step steps
    assert sum(1 for k, sh in meta["noise_log"] if sh[-2:] == [80, meta["frames"]]) == meta["K_fwd"] + 1
    assert np.array_equal(r["rq_codes"][0].numpy(), g["fwd_rq_codes"])
    for k in ("style", "pitch_pred", "decoder_inp", "coarse_mel"):
        assert _maxabs(r[k][0], g["fwd_" + k]) < TOL, k
    err = _maxabs(r["mel_out"][0], g["fwd_mel_out"])
    print(f"timesteps {meta['T_fwd']}, K_step {meta['K_fwd']}: oracle mel_out L-inf vs reference {err:.3e}")
    assert err < 5e-5


@pytest.mark.parametrize("key,K", [("smp", None), ("smp1", 1)])
def test_sampler_matches_reference(key, K):
    """(b) DiffusionDecoder.forward alone at timesteps 100, K_step 51; (d) the same at K_step 1 (one step, t = 0)."""
    g, meta = golden("ref_kstep")
    K = meta["K"] if K is None else K
    ns = O.NoiseSource(meta["seed"] + 2)
    with torch.no_grad():
        mel = O.mel_diffusion_sample(torch.from_numpy(g["smp_cond"])[None], torch.from_numpy(g["smp_coarse"])[None],
                                     acoustic_sd(), kstep_hp(meta["T"], K), ns)
    assert _log(ns) == meta[key + "_noise_log"] and len(ns.log) == K + 1
    err = _maxabs(mel[0], g[key + "_mel"])
    print(f"timesteps {meta['T']}, K_step {K}: sampler L-inf vs reference {err:.3e}")
    assert err < 5e-5


@pytest.mark.parametrize("interval", [10, 7])
def test_plms_matches_reference(interval):
    """(c) the pndm_speedup loop from t = K_step 51: t0 = 50 at interval 10, 49 at interval 7."""
    g, meta = golden("ref_kstep")
    assert meta[f"plms_i{interval}_t0"] == (meta["K"] - 1) // interval * interval
    ns = O.NoiseSource(meta["seed"] + 3)
    with torch.no_grad():
        mel = O.mel_diffusion_sample_plms(torch.from_numpy(g["smp_cond"])[None], torch.from_numpy(g["smp_coarse"])[None],
                                          acoustic_sd(), kstep_hp(meta["T"], meta["K"]), ns, interval)
    assert _log(ns) == meta[f"plms_i{interval}_noise_log"]
    ref = g[f"plms_i{interval}_mel"]
    err, scale = _maxabs(mel[0], ref), float(np.abs(ref).max())
    print(f"PLMS interval {interval}, K_step {meta['K']}: L-inf vs reference {err:.3e} (max |mel| {scale:.1f})")
    assert err < TOL * max(1.0, scale)


def test_k_step_equal_to_timesteps_is_the_oracle_bit_for_bit():
    """K_step = timesteps and an hp without K_step run the same samplers, bit for bit; a smaller K_step does not."""
    T, Fr = 12, 20
    gen = torch.Generator().manual_seed(3)
    cond = torch.randn(1, Fr, 256, generator=gen)
    coarse = (-3 + 0.8 * torch.randn(1, Fr, 80, generator=gen)).clamp(-6, 0.5)
    hp = kstep_hp(T, T)
    hp_nokey = {k: v for k, v in hp.items() if k != "K_step"}
    with torch.no_grad():
        a = O.mel_diffusion_sample(cond, coarse, acoustic_sd(), hp, O.NoiseSource(5))
        b = O.mel_diffusion_sample(cond, coarse, acoustic_sd(), hp_nokey, O.NoiseSource(5))
        p = O.mel_diffusion_sample_plms(cond, coarse, acoustic_sd(), hp, O.NoiseSource(6), 5)
        q = O.mel_diffusion_sample_plms(cond, coarse, acoustic_sd(), hp_nokey, O.NoiseSource(6), 5)
    assert torch.equal(a, b) and torch.equal(p, q)
    with torch.no_grad():  # and a smaller K does change the result
        d = O.mel_diffusion_sample(cond, coarse, acoustic_sd(), kstep_hp(T, T - 3), O.NoiseSource(5))
    assert not torch.equal(d, b)


@pytest.mark.parametrize("K", [1, 51, 100])
def test_resolve_accepts_k_step_up_to_timesteps(K):
    assert resolve(timesteps=100, K_step=K, f0_timesteps=100)["K_step"] == K
    if K > 1:  # PLMS intervals in [1, K_step)
        assert resolve(timesteps=100, K_step=K, pndm_speedup=K - 1)["pndm_speedup"] == K - 1


def test_resolve_prodiff_ignores_k_step():
    hp = resolve(decoder="prodiff", schedule_type="vpsde", timesteps=8, K_step=1000)
    assert hp["K_step"] == 1000


@pytest.mark.parametrize("kw", [dict(K_step=0), dict(K_step=-3), dict(K_step=101), dict(K_step=51, pndm_speedup=51),
                                dict(K_step=51, pndm_speedup=60), dict(K_step=1, pndm_speedup=1)])
def test_resolve_rejects_bad_k_step(kw):
    with pytest.raises(ValueError):
        resolve(timesteps=100, f0_timesteps=100, **kw)


def test_set_mel_k_step_is_exported():
    from stylesinger_b200._lib import lib
    assert lib.ssb_model_set_mel_k_step(None, 5) != 0 and "null model" in lib.ssb_last_error().decode()
