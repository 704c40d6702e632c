"""Padding through the CUDA path: padding phones (txt_tokens == 0), padding frames (mel2ph == 0) and padded reference mels
(ref_mels[:, 0] == 0), against the reference fixture ref_padded_T4 and the oracle, plus the key-masked branches of both
attention kernels against float64.  Every other GPU test leaves every mask all ones."""
import numpy as np
import pytest
import torch

from stylesinger_b200 import synth
from tests.common import (acoustic_engine, batch_noise, engine_noise_from_stream, golden, hp_for, oracle_forward,
                          utt_from_fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SCALE = 128 ** -0.5
T = 4


def _maxabs(a, b):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def _rel(a, b):
    """max |a - b| / max(1, max |b|): the bar for values that are not O(1)."""
    b = b.detach().cpu().double() if isinstance(b, torch.Tensor) else torch.as_tensor(np.asarray(b)).double()
    return _maxabs(a, b) / max(1.0, float(b.abs().max()))


# ---------------------------------------------------------------------------------------------------
# masked attention (engine.op_attention with a keymask) against float64
def _offsets(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


def _ref_attention(q, k, v, qo, ko, mask):
    out = torch.empty(q.shape[0], 256, dtype=torch.float64)
    for i in range(len(qo) - 1):
        qi, ki, vi = q[qo[i]:qo[i + 1]].double(), k[ko[i]:ko[i + 1]].double(), v[ko[i]:ko[i + 1]].double()
        keep = mask[ko[i]:ko[i + 1]] != 0
        for h in range(2):
            sl = slice(h * 128, (h + 1) * 128)
            s = (qi[:, sl] * SCALE) @ ki[:, sl].t()
            out[qo[i]:qo[i + 1], sl] = torch.softmax(s.masked_fill(~keep[None], float("-inf")), -1) @ vi[:, sl]
    return out


def _masked_case():
    """(query length, key length, mask over the keys) per utterance.  The guarded layout starts utterance b at a row
    congruent to k_offsets[b] mod 8, so the key lengths below give the wgmma kernel kshift > 0 from utterance 1 on."""
    def m(n, masked=(), valid=None):
        x = torch.ones(n)
        if valid is not None:
            x.zero_()
            x[list(valid)] = 1
        for a in masked:
            x[a] = 0
        return x
    cases = [
        (70, 37, m(37, [0])),                                             # key 0
        (1, 300, m(300, [63, 64, 127, 128])),                             # tile edges of the fp32 grid
        (200, 261, m(261, [slice(0, 70), slice(120, 200)])),              # a whole key tile of both grids at the front and one inside
        (129, 100, m(100, valid=[99])),                                   # only the last key
        (64, 151, m(151, valid=range(0, 151, 2))),                        # alternating
        (300, 90, m(90)),                                                 # nothing masked
        (5, 203, m(203, [slice(57, 71), slice(130, 203)])),               # kshift 3: the wgmma key tile edge at 61, a masked last tile
    ]
    return cases


def _qkv(ql, kl, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(int(sum(ql)), 256, generator=g) * 1.5
    k = torch.randn(int(sum(kl)), 256, generator=g) * 1.5
    v = torch.randn(int(sum(kl)), 256, generator=g)
    return q, k, v


@pytest.mark.parametrize("tc,bar", [(False, 2e-5), (True, 5e-5)])
def test_masked_attention_matches_float64(tc, bar):
    from stylesinger_b200.engine import op_attention
    cases = _masked_case()
    ql, kl = [c[0] for c in cases], [c[1] for c in cases]
    qo, ko = _offsets(ql), _offsets(kl)
    assert sorted(set(int(x) & 7 for x in ko[1:-1])) != [0]  # some key utterance starts off the 8-row grid
    q, k, v = _qkv(ql, kl, 31)
    mask = torch.cat([c[2] for c in cases])
    out = op_attention(q.to(DEV), k.to(DEV), v.to(DEV), qo, ko, SCALE, tc=tc, keymask=mask.to(DEV)).cpu()
    unmasked = op_attention(q.to(DEV), k.to(DEV), v.to(DEV), qo, ko, SCALE, tc=tc).cpu()
    ref = _ref_attention(q, k, v, qo, ko, mask)
    for i in range(len(cases)):
        rows = slice(int(qo[i]), int(qo[i + 1]))
        err = float((out[rows].double() - ref[rows]).abs().max())
        print(f"{'wgmma' if tc else 'fp32'} utterance {i} (q {ql[i]}, k {kl[i]}, kshift {int(ko[i]) & 7}): "
              f"L-inf vs float64 {err:.3e}")
        assert torch.isfinite(out[rows]).all() and err < bar, i
    # the mask matters wherever it masks something; the all-ones utterance equals the unmasked entry point bit for bit
    assert float((unmasked[qo[0]:qo[1]] - out[qo[0]:qo[1]]).abs().max()) > 100 * bar
    assert torch.equal(unmasked[qo[5]:qo[6]], out[qo[5]:qo[6]])


def test_fully_masked_utterance_is_nan_in_both_kernels_and_isolated():
    """An utterance whose keys are all masked, between two normal ones: both kernels write NaN for it (torch's softmax over
    all -inf does the same), and its neighbours are bit-identical to a batch without it.  Its key length is a multiple of
    8, so the third utterance keeps its place on the wgmma kernel's 8-row key grid."""
    from stylesinger_b200.engine import op_attention
    ql3, kl3 = [150, 77, 140], [203, 48, 333]
    q, k, v = _qkv(ql3, kl3, 32)
    mask = torch.ones(sum(kl3))
    mask[203:251] = 0
    mask[203 + 48 + 10] = 0  # and one ordinary masked key in the last utterance
    qo3, ko3 = _offsets(ql3), _offsets(kl3)
    keepq = torch.cat([torch.arange(0, 150), torch.arange(227, 367)])
    keepk = torch.cat([torch.arange(0, 203), torch.arange(251, 584)])
    qo2, ko2 = _offsets([150, 140]), _offsets([203, 333])
    ref = _ref_attention(q, k, v, qo3, ko3, mask)
    assert torch.isnan(ref[150:227]).all()
    outs = {}
    for tc in (False, True):
        o3 = op_attention(q.to(DEV), k.to(DEV), v.to(DEV), qo3, ko3, SCALE, tc=tc, keymask=mask.to(DEV)).cpu()
        o2 = op_attention(q[keepq].contiguous().to(DEV), k[keepk].contiguous().to(DEV), v[keepk].contiguous().to(DEV), qo2,
                          ko2, SCALE, tc=tc, keymask=mask[keepk].contiguous().to(DEV)).cpu()
        assert torch.isnan(o3[150:227]).all(), tc
        assert torch.equal(o3[keepq], o2), tc
        assert float((o3[keepq].double() - ref[keepq]).abs().max()) < (5e-5 if tc else 2e-5)
        outs[tc] = o3
    assert torch.isnan(outs[False][150:227]).all() and torch.isnan(outs[True][150:227]).all()


# ---------------------------------------------------------------------------------------------------
# the reference fixture through the CUDA forward
def _run_b1(m, u, seed, use_mel2ph=True, want=("style", "rq_codes", "pitch_pred", "decoder_inp", "coarse_mel",
                                                 "f0_denorm", "mel_out")):
    from stylesinger_b200.engine import pack_batch
    pb = pack_batch([u], use_mel2ph=use_mel2ph).to(DEV)
    if use_mel2ph:
        noise, _ = engine_noise_from_stream(seed, T, T, len(u["mel2ph"]), DEV)
        return m.forward(pb, noise=noise, want=want)
    dur, logdur = m.predict_durations(pb)
    F = int(dur.sum())
    pb.frame_offsets = np.array([0, F], np.int32)
    noise, _ = engine_noise_from_stream(seed, T, T, F, DEV)
    out = m.forward(pb, noise=noise, dur=dur, want=tuple(want) + ("mel2ph",))
    out["logdur"] = logdur
    return out


@pytest.mark.parametrize("denoiser_tc", [True, False])
def test_padded_fixture_matches_reference(denoiser_tc):
    g, meta = golden("ref_padded_T4")
    u = utt_from_fixture(g)
    m = acoustic_engine(T)
    try:
        m.set_tensor_cores(denoiser_tc)
        out = _run_b1(m, u, meta["seed"])
        dur = _run_b1(m, u, meta["seed"] + 1, use_mel2ph=False, want=("mel_out",))
    finally:
        m.set_tensor_cores(True)
    assert np.array_equal(out["rq_codes"].cpu().numpy().astype(np.int64), g["rq_codes"])
    errs = {k: _maxabs(out[k], g[k]) for k in ("style", "decoder_inp", "coarse_mel", "pitch_pred", "f0_denorm", "mel_out")}
    print("padded fixture, denoiser tc" if denoiser_tc else "padded fixture, denoiser FFMA", errs)
    for k in ("style", "decoder_inp", "coarse_mel", "pitch_pred"):
        assert errs[k] < 1e-4, k
    assert errs["f0_denorm"] < 5e-2  # Hz
    pad = g["in_mel2ph"] == 0
    assert (out["f0_denorm"].cpu().numpy()[pad] == 0).all()
    assert errs["mel_out"] < 1e-3
    assert np.array_equal(dur["mel2ph"].cpu().numpy().astype(np.int64), g["dur_mel2ph"])
    assert _maxabs(dur["logdur"], g["dur_logdur"][:, 0]) < 1e-4
    assert _maxabs(dur["mel_out"], g["dur_mel_out"]) < 1e-3


# ---------------------------------------------------------------------------------------------------
# a long padded utterance (wgmma decoder, decoder attention and aligner) and a ragged batch, against the oracle
def _with_padding(u, frame_runs=(), pad_phones=0, ref_tail=0, ref_col0_rows=()):
    u = {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in u.items()}
    for k in ("txt_tokens", "note", "note_type", "note_dur"):
        u[k] = torch.cat([u[k], torch.zeros(pad_phones, dtype=u[k].dtype)])
    for a, b in frame_runs:
        u["mel2ph"][a:b] = 0
    if ref_tail:
        u["ref_mels"][-ref_tail:] = 0
        u["ref_f0"][-ref_tail:] = 0
    for r in ref_col0_rows:
        u["ref_mels"][r, 0] = 0
    return u


def _long_padded():
    """1300 frames (11 row tiles): the decoder's FFT blocks, its attention and the style aligner take the wgmma kernels.
    70 leading padding frames mask the first key tile of both attention kernels; the interior run crosses the row tiles
    at 640 and 768 and masks the key tiles [640, 704) and [704, 768) whole."""
    u = synth.make_utterance(1300 / 187.5, utt_idx=105, ref_frames=200, frames=1300, phones=52)
    return _with_padding(u, frame_runs=[(0, 70), (630, 770), (1260, 1300)], pad_phones=4, ref_tail=20,
                         ref_col0_rows=(33,))


_ORACLE = {}


def _oracle(name, u, seed):
    if name not in _ORACLE:
        r, _ = oracle_forward(u, hp_for(T), seed)
        _ORACLE[name] = {k: v[0] for k, v in r.items() if isinstance(v, torch.Tensor) and v.dim() >= 1}
    return _ORACLE[name]


def _check_vs(out, ref, tag, fo=(0, None), ro=(0, None)):
    fs, rs = slice(*fo), slice(*ro)
    assert np.array_equal(out["rq_codes"][rs].cpu().numpy().astype(np.int64), ref["rq_codes"].cpu().numpy()), tag
    errs = {k: _rel(out[k][fs], ref[k]) for k in ("style", "decoder_inp", "coarse_mel", "pitch_pred")}
    errs["f0_denorm"] = _maxabs(out["f0_denorm"][fs], ref["f0_denorm"])
    errs["mel_out"] = _maxabs(out["mel_out"][fs], ref["mel_out"])
    print(tag, {k: f"{v:.2e}" for k, v in errs.items()})
    for k in ("style", "decoder_inp", "coarse_mel", "pitch_pred"):
        assert errs[k] < 1e-4, (tag, k)
    assert errs["f0_denorm"] < 5e-2, tag
    assert errs["mel_out"] < 1e-3, tag


WANT = ("style", "rq_codes", "pitch_pred", "decoder_inp", "coarse_mel", "f0_denorm", "mel_out")


def test_long_padded_utterance_matches_oracle_on_both_kernel_paths():
    from stylesinger_b200._lib import lib
    u = _long_padded()
    m = acoustic_engine(T)
    ref = _oracle("long", u, 410)
    on = _run_b1(m, u, 410)
    on = {k: v.clone() for k, v in on.items()}
    _check_vs(on, ref, "long padded, wgmma")
    pad = (u["mel2ph"] == 0).numpy()
    assert (on["f0_denorm"].cpu().numpy()[pad] == 0).all()
    try:
        m.set_fft_tensor_cores(False)
        lib.ssb_set_attention_tensor_cores(0)
        off = _run_b1(m, u, 410)
    finally:
        m.set_fft_tensor_cores(True)
        lib.ssb_set_attention_tensor_cores(1)
    for k in ("style", "decoder_inp", "coarse_mel", "pitch_pred", "mel_out"):
        e = _rel(on[k], off[k])
        print(f"long padded {k}: wgmma vs fp32 kernels {e:.2e}")
        assert e < 1e-4, k
    assert torch.equal(on["rq_codes"], off["rq_codes"])


def test_ragged_padded_batch_matches_oracle_and_solo_runs():
    """The fixture utterance, an unpadded one, the long padded one and one whose only padding is in its reference mel.
    Inside the batch every utterance takes the wgmma attention; the short ones take the fp32 kernel when run alone."""
    from stylesinger_b200.engine import pack_batch
    g, meta = golden("ref_padded_T4")
    plain = synth.make_utterance(90 / 187.5, utt_idx=106, ref_frames=40, frames=90, phones=9)
    refpad = _with_padding(synth.make_utterance(70 / 187.5, utt_idx=107, ref_frames=60, frames=70, phones=7),
                           ref_tail=13, ref_col0_rows=(5, 30))
    utts = [("fixture", utt_from_fixture(g), meta["seed"]), ("plain", plain, 420), ("long", _long_padded(), 410),
            ("refpad", refpad, 430)]
    m = acoustic_engine(T)
    pb = pack_batch([u for _, u, _ in utts]).to(DEV)
    per = [engine_noise_from_stream(s, T, T, len(u["mel2ph"]), DEV)[0] for _, u, s in utts]
    out = m.forward(pb, noise=batch_noise(per), want=WANT)
    out = {k: v.clone() for k, v in out.items()}
    fo, ro = pb.frame_offsets, pb.ref_offsets
    for i, (name, u, seed) in enumerate(utts):
        f, r = (int(fo[i]), int(fo[i + 1])), (int(ro[i]), int(ro[i + 1]))
        _check_vs(out, _oracle(name, u, seed), f"batch[{name}] vs oracle", f, r)
        solo = _run_b1(m, u, seed)
        _check_vs(out, solo, f"batch[{name}] vs solo", f, r)
