"""GPU parity tests: the CUDA path (through the C ABI) against the oracle and the reference-generated
golden fixtures.  Tolerances: the hot path computes in fp32 (FFMA); the stated bar is mel L-inf < 1e-3
(BASELINE.json); per-operator checks are much tighter.  Integer paths (RVQ codes, mel2ph) are bit-exact.
"""
import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG
from tests.common import (acoustic_engine, acoustic_sd, batch_noise, engine_noise_from_stream, golden, hp_for,
                          oracle_forward, utt_from_meta, vocoder_engine, vocoder_sd)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _maxabs(a, b):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


# ---------------------------------------------------------------------------------------------------
def test_denoisers_match_reference_golden():
    g, meta = golden("ref_small_T4")
    m = acoustic_engine(meta["T"])
    Fr = g["dn_spec"].shape[1]
    offs = np.array([0, Fr], np.int32)
    cond = torch.from_numpy(g["dn_cond"].T.copy()).to(DEV)
    e = m.denoiser_eval(0, torch.from_numpy(g["dn_spec"].T.copy()).to(DEV), None, meta["T"] - 1, cond, offs)
    assert _maxabs(e.cpu().numpy().T, g["dn_out"]) < 5e-5
    f0 = torch.from_numpy(g["dd_f0"]).to(DEV)
    uv = torch.from_numpy(g["dd_uv"].astype(np.int32)).to(DEV)
    e2 = m.denoiser_eval(1, f0, uv, 1, cond, offs)
    e3 = m.denoiser_eval(2, f0, uv, 0, cond, offs)
    assert _maxabs(e2.cpu().numpy().T, g["dd_out"]) < 5e-5
    assert _maxabs(e3.cpu().numpy().T, g["dd_out_inp"]) < 5e-5


def test_rvq_codes_bit_exact_vs_reference_golden():
    g, meta = golden("ref_small_T4")
    m = acoustic_engine(meta["T"])
    # the fixture is stored Fortran-ordered (the reference's tensor is a transposed view): make it row-major
    x = torch.from_numpy(np.ascontiguousarray(g["rq_in"])).to(DEV)
    with pytest.raises(ValueError):
        m.rvq(torch.from_numpy(g["rq_in"]).to(DEV), np.array([0, x.shape[0]], np.int32))  # strided view: refused
    q, codes = m.rvq(x, np.array([0, x.shape[0]], np.int32))
    assert np.array_equal(codes.cpu().numpy().astype(np.int64), g["rq_codes"])
    with torch.no_grad():
        qo, _ = O.rq_quantize(torch.from_numpy(g["rq_in"])[None], acoustic_sd())
    assert _maxabs(q, qo[0]) < 1e-6


def test_rvq_codes_bit_exact_on_random_vectors():
    m = acoustic_engine(4)
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(3000, 256, generator=gen) * 1.5
    q, codes = m.rvq(x.to(DEV), np.array([0, 1000, 1001, 3000], np.int32))
    with torch.no_grad():
        qo, co = O.rq_quantize(x[None], acoustic_sd())
    assert np.array_equal(codes.cpu().numpy().astype(np.int64), co[0].numpy())
    assert _maxabs(q, qo[0]) < 1e-6


def _run_engine_b1(meta, T, seed, use_mel2ph=True, want=None):
    from stylesinger_b200.engine import pack_batch
    u = utt_from_meta(meta)
    m = acoustic_engine(T)
    pb = pack_batch([u], use_mel2ph=use_mel2ph).to(DEV)
    want = want or ("mel_out", "f0_denorm", "style", "rq_codes", "pitch_pred", "decoder_inp", "coarse_mel", "encoder_out")
    if not use_mel2ph:
        dur, logdur = m.predict_durations(pb)
        d = dur.cpu().numpy()
        pb.frame_offsets = np.array([0, int(d.sum())], np.int32)
        noise, _ = engine_noise_from_stream(seed, T, T, int(d.sum()), DEV)
        out = m.forward(pb, noise=noise, dur=dur, want=tuple(want) + ("mel2ph",))
        out["logdur"] = logdur
        return out
    noise, _ = engine_noise_from_stream(seed, T, T, meta["frames"], DEV)
    return m.forward(pb, noise=noise, want=want)


def test_full_forward_T4_matches_reference_golden():
    g, meta = golden("ref_small_T4")
    out = _run_engine_b1(meta, meta["T"], meta["seed"])
    assert np.array_equal(out["rq_codes"].cpu().numpy().astype(np.int64), g["rq_codes"])  # bit-exact
    assert _maxabs(out["style"], g["style"]) < 1e-4
    assert _maxabs(out["pitch_pred"], g["pitch_pred"]) < 1e-4
    assert _maxabs(out["decoder_inp"], g["decoder_inp"]) < 1e-4
    assert _maxabs(out["coarse_mel"], g["coarse_mel"]) < 1e-4
    assert _maxabs(out["f0_denorm"], g["f0_denorm"]) < 5e-2  # Hz
    assert _maxabs(out["mel_out"], g["mel_out"]) < 1e-3  # the BASELINE.json bar; observed ~1e-5


def test_duration_path_matches_reference_golden():
    g, meta = golden("ref_small_T4")
    out = _run_engine_b1(meta, meta["T"], meta["seed"] + 1, use_mel2ph=False)
    assert np.array_equal(out["mel2ph"].cpu().numpy().astype(np.int64), g["dur_mel2ph"])  # integer path: exact
    assert _maxabs(out["logdur"], g["dur_logdur"][:, 0]) < 1e-4
    assert _maxabs(out["mel_out"], g["dur_mel_out"]) < 1e-3


def test_T25_matches_reference_golden():
    g, meta = golden("ref_f64_T25")
    out = _run_engine_b1(meta, meta["T"], meta["seed"])
    assert np.array_equal(out["rq_codes"].cpu().numpy().astype(np.int64), g["rq_codes"])
    assert _maxabs(out["pitch_pred"], g["pitch_pred"]) < 1e-4
    assert _maxabs(out["mel_out"], g["mel_out"]) < 1e-3


def test_ragged_batch_equals_b1_oracle():
    """True-length semantics: every utterance of a ragged batch matches its own B=1 oracle run."""
    from stylesinger_b200 import synth
    from stylesinger_b200.engine import pack_batch
    T = 4
    hp = hp_for(T)
    specs = [(40, 6, 50, 200), (150, 14, 33, 201), (97, 9, 80, 202)]
    utts = [synth.make_utterance(f / 187.5, utt_idx=i, ref_frames=r, frames=f, phones=p) for f, p, r, i in specs]
    m = acoustic_engine(T)
    pb = pack_batch(utts).to(DEV)
    per = [engine_noise_from_stream(300 + i, T, T, u["mel2ph"].shape[0], DEV)[0] for i, u in enumerate(utts)]
    out = m.forward(pb, noise=batch_noise(per), want=("mel_out", "f0_denorm", "rq_codes", "style"))
    fo, ro = pb.frame_offsets, pb.ref_offsets
    for i, u in enumerate(utts):
        r, _ = oracle_forward(u, hp, 300 + i)
        assert np.array_equal(out["rq_codes"][ro[i]:ro[i + 1]].cpu().numpy().astype(np.int64), r["rq_codes"][0].numpy())
        assert _maxabs(out["style"][fo[i]:fo[i + 1]], r["style"][0]) < 1e-4
        assert _maxabs(out["mel_out"][fo[i]:fo[i + 1]], r["mel_out"][0]) < 1e-3


def test_mel_diffusion_T100_vs_oracle():
    """Config-2 style check at reduced length: 100 sampler steps with injected noise, mel L-inf < 1e-3."""
    T, Fr = 100, 80
    hp = hp_for(T)
    gen = torch.Generator().manual_seed(77)
    cond = torch.randn(1, Fr, 256, generator=gen)
    coarse = (-3 + 0.8 * torch.randn(1, Fr, 80, generator=gen)).clamp(-6, 0.5)
    ns = O.NoiseSource(123)
    ns.record = []
    with torch.no_grad():
        ref = O.mel_diffusion_sample(cond, coarse, acoustic_sd(), hp, ns)
    noise = torch.stack([n[0, 0].t().contiguous() for n in ns.record]).contiguous().to(DEV)
    m = acoustic_engine(T, 4)
    mel = m.mel_diffusion(cond[0].to(DEV).contiguous(), coarse[0].to(DEV).contiguous(), np.array([0, Fr], np.int32), noise)
    err = _maxabs(mel, ref[0])
    print("mel L-inf after T=100:", err)
    assert err < 1e-3


def test_f0_diffusion_vs_oracle():
    T, Fr = 12, 90
    hp = hp_for(4, T)
    gen = torch.Generator().manual_seed(78)
    cond = torch.randn(1, 256, Fr, generator=gen)
    midi = torch.randint(50, 70, (1, 1, Fr), generator=gen).float()
    lo, hi = O.midi_clip_band(midi)
    ns = O.NoiseSource(321)
    ns.record = []
    with torch.no_grad():
        ref = O.f0_diffusion_sample(cond, (lo, hi), acoustic_sd(), hp, "gm_diffnet_inpainte.", ns)
    rec = ns.record
    g = torch.stack([rec[1].reshape(Fr)] + [rec[2 + 2 * i].reshape(Fr) for i in range(T)]).contiguous().to(DEV)
    u = torch.stack([rec[3 + 2 * i][0].t().contiguous() for i in range(T)]).contiguous().to(DEV)
    m = acoustic_engine(4, T)
    z, uv = m.f0_diffusion(1, cond[0].t().contiguous().to(DEV), lo.reshape(Fr).to(DEV), hi.reshape(Fr).to(DEV),
                           np.array([0, Fr], np.int32), g, u)
    flips = int((uv.cpu().numpy() != ref[0, :, 1].numpy().astype(np.int32)).sum())
    assert flips == 0, flips
    assert _maxabs(z, ref[0, :, 0]) < 1e-4


# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tc", [True, False])
def test_vocoder_matches_reference_golden(tc):
    g, meta = golden("ref_vocoder_f24")
    v = vocoder_engine()
    v.set_tensor_cores(tc)
    Fr = g["mel"].shape[0]
    ns = O.NoiseSource(meta["seed"] + 5)
    ini = ns.rand((1, 9))
    ini[:, 0] = 0
    src = ns.randn((1, Fr * 256, 9))[0].contiguous()
    offs = np.array([0, Fr], np.int32)
    wav = v.generate(torch.from_numpy(g["mel"]).to(DEV), torch.from_numpy(g["f0"]).to(DEV), offs,
                     rand_ini=ini.to(DEV).contiguous(), src_noise=src.to(DEV))
    err = _maxabs(wav, g["wav"])
    print("wav L-inf:", err)
    assert err < 1e-3
    wav2 = v.generate(torch.from_numpy(g["mel"]).to(DEV), None, offs)
    err2 = _maxabs(wav2, g["wav_nof0"])
    print("tc" if tc else "simt", "wav L-inf:", err, "no-f0:", err2)
    v.set_tensor_cores(True)
    assert err2 < 1e-3


def test_vocoder_ragged_batch_equals_b1_oracle():
    v = vocoder_engine()
    gen = torch.Generator().manual_seed(9)
    lens = [17, 40]
    mels, f0s, refs, inis, srcs = [], [], [], [], []
    for i, Fr in enumerate(lens):
        mel = (-3.0 + 0.8 * torch.randn(Fr, 80, generator=gen)).clamp(-6, 1.5)
        f0 = 150 + 350 * torch.rand(Fr, generator=gen)
        f0[2:5] = 0
        ns = O.NoiseSource(50 + i)
        ns.record = []
        with torch.no_grad():
            refs.append(O.spec2wav(mel.numpy(), f0.numpy(), vocoder_sd(), DEFAULT_VOCODER_CONFIG, ns))
        ini = ns.record[0].clone()
        ini[:, 0] = 0
        inis.append(ini[0])
        srcs.append(ns.record[1][0])
        mels.append(mel)
        f0s.append(f0)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    wav = v.generate(torch.cat(mels).to(DEV), torch.cat(f0s).to(DEV), offs, rand_ini=torch.stack(inis).contiguous().to(DEV),
                     src_noise=torch.cat(srcs).contiguous().to(DEV)).cpu().numpy()
    for i in range(2):
        assert _maxabs(wav[offs[i] * 256:offs[i + 1] * 256], refs[i]) < 1e-3


def test_philox_mode_runs_and_is_deterministic():
    from stylesinger_b200.engine import pack_batch
    g, meta = golden("ref_small_T4")
    u = utt_from_meta(meta)
    m = acoustic_engine(4)
    pb = pack_batch([u]).to(DEV)
    a = m.forward(pb, noise=None, seed=7)["mel_out"].clone()
    b = m.forward(pb, noise=None, seed=7)["mel_out"].clone()
    c = m.forward(pb, noise=None, seed=8)["mel_out"].clone()
    assert torch.isfinite(a).all()
    assert torch.equal(a, b) and not torch.equal(a, c)
