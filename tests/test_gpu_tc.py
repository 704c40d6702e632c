"""wgmma path (fp16 hi/lo split operands, 3 MMAs per product, fp32 register accumulators) against torch fp32
and against the reference-generated goldens; and SIMT-vs-tensor-core agreement of the samplers."""
import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from tests.common import acoustic_engine, acoustic_sd, golden, hp_for

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _maxabs(a, b):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def test_denoiser_large_batch_pair_kernel_matches_simt():
    """DiffNet / DDiffNet evaluation on ~20k frames (CTA-pair kernel territory) against the fp32 FFMA path."""
    T = 4
    m = acoustic_engine(T)
    gen = torch.Generator().manual_seed(3)
    lens = [2900, 1700, 2999, 800, 2300, 1950, 2450, 3000, 1300, 1111]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    n = int(offs[-1])
    cond = torch.randn(n, 256, generator=gen).to(DEV)
    spec = torch.randn(n, 80, generator=gen).to(DEV)
    f0 = torch.randn(n, generator=gen).to(DEV)
    uv = (torch.rand(n, generator=gen) > 0.5).to(torch.int32).to(DEV)
    out = {}
    try:
        for tc in (True, False):
            m.set_tensor_cores(tc)
            out[tc] = (m.denoiser_eval(0, spec, None, 2, cond, offs).clone(), m.denoiser_eval(1, f0, uv, 1, cond, offs).clone())
    finally:
        m.set_tensor_cores(True)
    errs = (_maxabs(out[True][0], out[False][0]), _maxabs(out[True][1], out[False][1]))
    print("pair-kernel denoisers vs simt:", errs)
    assert max(errs) < 1e-4


@pytest.mark.parametrize("tc", [True, False])
def test_denoisers_match_reference_golden(tc):
    g, meta = golden("ref_small_T4")
    m = acoustic_engine(meta["T"])
    assert m.set_tensor_cores(tc) == tc
    try:
        Fr = g["dn_spec"].shape[1]
        offs = np.array([0, Fr], np.int32)
        cond = torch.from_numpy(g["dn_cond"].T.copy()).to(DEV)
        e = m.denoiser_eval(0, torch.from_numpy(g["dn_spec"].T.copy()).to(DEV), None, meta["T"] - 1, cond, offs)
        f0 = torch.from_numpy(g["dd_f0"]).to(DEV)
        uv = torch.from_numpy(g["dd_uv"].astype(np.int32)).to(DEV)
        e2 = m.denoiser_eval(1, f0, uv, 1, cond, offs)
        e3 = m.denoiser_eval(2, f0, uv, 0, cond, offs)
        errs = (_maxabs(e.cpu().numpy().T, g["dn_out"]), _maxabs(e2.cpu().numpy().T, g["dd_out"]),
                _maxabs(e3.cpu().numpy().T, g["dd_out_inp"]))
        print("tc" if tc else "simt", "denoiser errs", errs)
        assert max(errs) < 5e-5
    finally:
        m.set_tensor_cores(True)


@pytest.mark.parametrize("mode", ["persistent", "per_launch_tc", "simt"])
def test_mel_diffusion_T100_vs_oracle(mode):
    """T=100 reverse steps with injected noise: single-launch persistent wgmma kernel, one launch per GEMM
    (wgmma), and the fp32 FFMA path all stay far below the mel L-inf < 1e-3 bar."""
    T, Fr = 100, 200
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
    m.set_tensor_cores(mode != "simt")
    m.set_persistent(mode == "persistent")
    try:
        mel = m.mel_diffusion(cond[0].to(DEV).contiguous(), coarse[0].to(DEV).contiguous(), np.array([0, Fr], np.int32), noise)
        err = _maxabs(mel, ref[0])
        print(mode, "mel L-inf after T=100:", err)
        assert err < 1e-3
    finally:
        m.set_tensor_cores(True)
        m.set_persistent(True)


def test_persistent_matches_per_launch_on_ragged_batch_philox():
    """Same Philox streams in both paths: a ragged 3-utterance batch must agree to fp32 rounding."""
    T = 20
    m = acoustic_engine(T, 4)
    gen = torch.Generator().manual_seed(5)
    lens = [130, 257, 64]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    cond = torch.randn(int(offs[-1]), 256, generator=gen).to(DEV)
    coarse = (-3 + 0.8 * torch.randn(int(offs[-1]), 80, generator=gen)).clamp(-6, 0.5).to(DEV)
    try:
        m.set_persistent(True)
        a = m.mel_diffusion(cond, coarse, offs, None, seed=9).clone()
        m.set_persistent(False)
        b = m.mel_diffusion(cond, coarse, offs, None, seed=9).clone()
    finally:
        m.set_persistent(True)
    err = _maxabs(a, b)
    print("persistent vs per-launch (philox, ragged):", err)
    assert torch.isfinite(a).all() and err < 1e-3


def test_f0_pair_persistent_matches_oracle_and_per_launch():
    """Full forward (T=12 F0 steps, mel diffusion skipped) with injected noise: the persistent two-net F0 sampler
    vs the per-launch path vs the oracle (pitch_pred, f0_denorm; UV decisions must not flip)."""
    from stylesinger_b200 import synth
    from stylesinger_b200.engine import pack_batch
    from tests.common import engine_noise_from_stream, oracle_forward
    T = 12
    hp = hp_for(T)
    u = synth.make_utterance(150 / 187.5, utt_idx=321, ref_frames=40, frames=150, phones=11)
    r, _ = oracle_forward(u, hp, 555, skip_diffusion=True)
    m = acoustic_engine(T)
    pb = pack_batch([u]).to(DEV)
    outs = {}
    try:
        for mode in ("persistent", "per_launch"):
            m.set_persistent(mode == "persistent")
            noise, _ = engine_noise_from_stream(555, T, T, 150, DEV)
            outs[mode] = m.forward(pb, noise=noise, skip_mel_diffusion=True, want=("pitch_pred", "f0_denorm", "decoder_inp"))
            for k in ("pitch_pred", "f0_denorm"):
                outs[mode][k] = outs[mode][k].clone()
    finally:
        m.set_persistent(True)
    for mode, o in outs.items():
        e_pp = _maxabs(o["pitch_pred"], r["pitch_pred"][0])
        e_f0 = _maxabs(o["f0_denorm"], r["f0_denorm"][0])
        print(mode, "pitch_pred err", e_pp, "f0_denorm err (Hz)", e_f0)
        assert e_pp < 1e-3 and e_f0 < 0.5


def test_decoder_fft_ffn_tensor_cores_match_ffma():
    """A 12 s utterance (2250 frames) puts the decoder's GEMMs (QKV / out projections, FFN conv k=9 -> gelu -> linear) and
    the style aligner's five projections per layer on the wgmma kernel; the same pass with that switch off keeps them on
    the fp32 FFMA kernel.  Same Philox streams, so style / decoder_inp / coarse_mel must agree to fp32 rounding."""
    from stylesinger_b200 import synth
    from stylesinger_b200.engine import pack_batch
    T = 4
    u = synth.make_utterance(12.0, utt_idx=77)
    m = acoustic_engine(T)
    pb = pack_batch([u]).to(DEV)
    out, ran = {}, {}
    from stylesinger_b200._lib import variant_launches
    try:
        for on in (True, False):
            assert m.set_fft_tensor_cores(on) == on
            before = variant_launches()
            o = m.forward(pb, seed=11, skip_mel_diffusion=True, want=("decoder_inp", "coarse_mel", "style"))
            after = variant_launches()
            ran[on] = {k: v - before.get(k, 0) for k, v in after.items() if "GENERIC" in k and v - before.get(k, 0) > 0}
            out[on] = {k: v.clone() for k, v in o.items()}
    finally:
        m.set_fft_tensor_cores(True)
    # 2 aligner layers x 5 projections + 4 decoder layers x (qkv, out, ffn1, ffn2) GENERIC wgmma GEMMs more than with the switch off
    assert sum(ran[True].values()) - sum(ran[False].values()) == 2 * 5 + 4 * 4, ran
    for k in ("style", "decoder_inp"):
        e = _maxabs(out[True][k], out[False][k])
        sc = float(out[False][k].abs().max())
        print(f"{k}: wgmma vs FFMA max |diff| {e:.3e} (max |value| {sc:.2f})")
        assert e < 1e-4 * max(1.0, sc), k
    err = _maxabs(out[True]["coarse_mel"], out[False]["coarse_mel"])
    scale = float(out[False]["coarse_mel"].abs().max())
    print(f"decoder FFN wgmma vs FFMA: coarse_mel max |diff| {err:.3e} (max |value| {scale:.2f})")
    assert err < 1e-4 * max(1.0, scale)


ATTN_TC_DEFAULT = 1  # library default of the switch (csrc/attention_tc.cu attention_tc_enabled)


def test_forward_attention_tensor_cores_match_fp32_kernel():
    """Same 12 s forward with the decoder's self-attention and the aligner's cross-attention on the wgmma kernel vs the
    fp32 kernel (all projections on wgmma both times): style / decoder_inp / coarse_mel agree to fp32 rounding."""
    from stylesinger_b200 import synth
    from stylesinger_b200._lib import lib
    from stylesinger_b200.engine import pack_batch
    u = synth.make_utterance(12.0, utt_idx=78)
    m = acoustic_engine(4)
    pb = pack_batch([u]).to(DEV)
    out = {}
    try:
        for on in (True, False):
            lib.ssb_set_attention_tensor_cores(1 if on else 0)
            l0 = lib.ssb_launch_count()
            o = m.forward(pb, seed=12, skip_mel_diffusion=True, want=("decoder_inp", "coarse_mel", "style"))
            out[on] = {k: v.clone() for k, v in o.items()}
            out[on]["launches"] = lib.ssb_launch_count() - l0
    finally:
        lib.ssb_set_attention_tensor_cores(ATTN_TC_DEFAULT)
    for k in ("style", "decoder_inp", "coarse_mel"):
        e = _maxabs(out[True][k], out[False][k])
        sc = float(out[False][k].abs().max())
        print(f"{k}: attention wgmma vs fp32 kernel max |diff| {e:.3e} (max |value| {sc:.2f})")
        assert torch.isfinite(out[True][k]).all() and e < 1e-4 * max(1.0, sc), k


def test_two_model_handles_on_two_streams_match_sequential():
    """Two model handles driving CTA-pair (cluster) GEMMs from two torch streams at once: both streams must drain and
    reproduce the sequential results bit for bit."""
    from stylesinger_b200.engine import AcousticModel
    from stylesinger_b200._lib import variant_launches
    T = 6
    lens = [2900, 1700, 2999, 800, 2300, 1950, 2450, 3000, 1300, 1111]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    n = int(offs[-1])
    g = torch.Generator().manual_seed(21)
    cond = torch.randn(n, 256, generator=g).to(DEV)
    lo, hi = torch.full((n,), -1.0, device=DEV), torch.full((n,), 1.0, device=DEV)
    models = [AcousticModel(acoustic_sd(), hp_for(4, T)) for _ in range(2)]
    seq = [m.f0_diffusion(i, cond, lo, hi, offs, seed=30 + i) for i, m in enumerate(models)]
    seq = [(z.clone(), uv.clone()) for z, uv in seq]
    torch.cuda.synchronize()
    before = variant_launches()
    streams = [torch.cuda.Stream(device=DEV) for _ in range(2)]
    outs = [None, None]
    for rep in range(3):
        for i, (m, st) in enumerate(zip(models, streams)):
            with torch.cuda.stream(st):
                z, uv = m.f0_diffusion(i, cond, lo, hi, offs, seed=30 + i)
                outs[i] = (z.clone(), uv.clone())
    torch.cuda.synchronize()
    after = variant_launches()
    ran = {k: v - before.get(k, 0) for k, v in after.items() if v - before.get(k, 0) > 0}
    assert any(k.startswith("tc2") for k in ran), ran  # CTA-pair kernels were in flight from both streams
    for i in range(2):
        assert torch.equal(outs[i][0], seq[i][0]) and torch.equal(outs[i][1], seq[i][1])
