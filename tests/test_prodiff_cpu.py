"""ProDiff teacher mel decoder (hparams['decoder'] == 'prodiff'), CPU side: the product's schedule table, the test oracle's
restatement and the synthetic checkpoint against the unmodified reference (tests/golden/ref_prodiff_T8.npz), the
hparams rules, and the C ABI's mode check (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200.hparams import resolve
from stylesinger_b200.schedules import prodiff_schedule, prodiff_table
from tests.common import golden, prodiff_hp, prodiff_sd, utt_from_meta

TOL = 2e-5  # fp32 CPU, same op order up to BLAS blocking (as tests/test_oracle_golden.py)
COMMENTED_CONFIG = {"timesteps": 8, "timescale": 1, "K_step": 1000, "schedule_type": "vpsde", "max_beta": 0.06,
                    "pndm_speedup": 10, "residual_layers": 20, "residual_channels": 256, "dilation_cycle_length": 4}


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def test_prodiff_table_matches_reference_buffers():
    g, meta = golden("ref_prodiff_T8")
    T = meta["T"]
    s, o = prodiff_schedule(T), O.prodiff_tables(T)
    for k in s:
        ref = g["sched_" + k]
        assert ref.shape == (T + 1,)
        assert np.array_equal(s[k], ref), (k, "product")
        assert np.array_equal(o[k].numpy(), ref), (k, "oracle")
    tab = prodiff_table(T)
    assert tab.shape == (T, 8) and tab.dtype == np.float32
    assert np.all(tab[:, 0] == 0) and np.all(tab[:, 1] == -1)
    assert np.array_equal(tab[:, 2], g["sched_posterior_mean_coef1"][:T])
    assert np.array_equal(tab[:, 3], g["sched_posterior_mean_coef2"][:T])
    assert np.array_equal(tab[:, 7], g["sched_alphas_cumprod"][:T])
    sig = (0.5 * torch.from_numpy(g["sched_posterior_log_variance_clipped"][:T])).exp().numpy()  # the reference's fp32 op
    assert tab[0, 4] == 0 and np.allclose(tab[1:, 4], sig[1:], rtol=2e-7, atol=0)
    print("betas[0]", float(g["sched_betas"][0]), "max |sigma - ref|", _maxabs(tab[1:, 4], sig[1:]))


def test_oracle_prodiff_sampler_matches_reference():
    g, meta = golden("ref_prodiff_T8")
    hp = prodiff_hp()
    ns = O.NoiseSource(meta["sampler_seed"])
    with torch.no_grad():
        mel = O.mel_prodiff_sample(torch.from_numpy(g["sampler_cond"])[None], prodiff_sd(), hp, ns)
    assert [[k, list(sh)] for k, sh in ns.log] == meta["sampler_noise_log"]
    err, scale = _maxabs(mel[0].numpy(), g["sampler_mel"]), float(np.abs(g["sampler_mel"]).max())
    print("oracle ProDiff sampler L-inf:", err, "|mel|max:", scale)
    assert err < TOL * max(1.0, scale), (err, scale)


def test_oracle_prodiff_forward_matches_reference():
    g, meta = golden("ref_prodiff_T8")
    hp = prodiff_hp()
    u = utt_from_meta(meta)
    ns = O.NoiseSource(meta["seed"])
    with torch.no_grad():
        r = O.stylesinger_forward(prodiff_sd(), hp, u["txt_tokens"][None], u["note"][None], u["note_dur"][None],
                                  u["note_type"][None], u["spk_embed"][None], u["emo_embed"][None], u["ref_mels"][None],
                                  u["ref_f0"], ns, mel2ph=u["mel2ph"][None])
    assert [[k, list(sh)] for k, sh in ns.log] == meta["noise_log"]
    e_dec = _maxabs(r["decoder_inp"][0].numpy(), g["decoder_inp"])
    e_f0 = _maxabs(r["f0_denorm"][0].numpy(), g["f0_denorm"])
    e_mel, scale = _maxabs(r["mel_out"][0].numpy(), g["mel_out"]), float(np.abs(g["mel_out"]).max())
    print("oracle ProDiff forward L-inf: decoder_inp", e_dec, "f0_denorm(Hz)", e_f0, "mel_out", e_mel, "|mel|max", scale)
    assert e_dec < TOL
    assert e_f0 < 1e-3
    assert e_mel < TOL * max(1.0, scale)


def test_synth_prodiff_state_dict_has_the_reference_keys_and_shapes():
    g, meta = golden("ref_prodiff_T8")
    sd = prodiff_sd()
    ours = [[k, list(v.shape)] for k, v in sd.items()]
    assert ours == meta["state_dict"]
    assert not any(k.startswith(("postdiff.", "ln_proj.")) for k in sd)
    assert sd["diff_decoder.timesteps"].dim() == 0 and float(sd["diff_decoder.timesteps"]) == meta["T"]


def test_commented_config_resolves():
    """The ProDiff block of egs/stylesinger.yaml:145-155, K_step 1000 and pndm_speedup 10 included: accepted and ignored
    by the ProDiff path, as the reference ignores them."""
    hp = resolve(dict(COMMENTED_CONFIG, decoder="prodiff"))
    assert hp["decoder"] == "prodiff" and hp["K_step"] == 1000 and hp["pndm_speedup"] == 10
    with pytest.raises(NotImplementedError):  # the same keys stay refused for the DiffSinger decoder
        resolve(dict(COMMENTED_CONFIG))
    with pytest.raises(ValueError):  # (PLMS interval 10 at T = 8)
        resolve(dict(COMMENTED_CONFIG, schedule_type="linear"))


def test_prodiff_with_another_schedule_type_raises():
    with pytest.raises(NotImplementedError):
        resolve(decoder="prodiff", schedule_type="linear")
    with pytest.raises(NotImplementedError):
        prodiff_table(8, "linear")
    with pytest.raises(NotImplementedError):
        resolve(decoder="fft")


def test_model_create_ex_rejects_an_unknown_mode_without_a_gpu():
    from stylesinger_b200._lib import HParams, lib
    h = C.c_void_p()
    rc = lib.ssb_model_create_ex(C.byref(h), None, 0, C.byref(HParams()), 7)
    msg = lib.ssb_last_error().decode()
    print("rc", rc, "message:", msg)
    assert rc != 0 and not h.value
    assert "unknown mel_decoder 7" in msg
