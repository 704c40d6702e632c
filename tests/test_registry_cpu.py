"""The per-registry drop-ins (FS_ENCODERS['fft'], FS_DECODERS['fft'], StyleSinger.get_style, the denoisers) on the CPU.

1. The float64 oracle computes the function the reference computes: it agrees with the reference fixtures within the fp32
   oracle's own bar.  The GPU tests (tests/test_gpu_fft_style.py) measure the CUDA path against it.
2. The oracle against ref_registry, written by the unmodified reference's FastspeechEncoder / FastspeechDecoder on padded
   B = 3 batches and by its get_style at B = 1 (tools/make_golden.py registry).
3. The host logic of the facades in stylesinger_b200/modules.py with a stand-in engine: the length rule (the index after
   the last non-padding row, never a count of them), padded <-> packed conversion and the denoiser layouts.
"""
import numpy as np
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import modules as M
from tests.common import (acoustic_sd, acoustic_sd64, golden, hp_for, registry_inputs, utt_from_fixture,
                          utt_from_meta)

TOL = 2e-5  # the fp32 oracle's bar against the reference (tests/test_oracle_golden.py)


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


# ---------------------------------------------------------------------------------------------------------------------
# 1. float64 oracle vs the reference fixtures of the full forward
def _forward64(u, g, hp):
    """The deterministic half of a B = 1 forward on the float64 state dict (stylesinger.py:119-187): encoder, duration
    predictor, expansion, get_style, pitch embedding, FFT decoder and mel_out, with the reference's own RVQ codes and F0
    (an argmin and a sampler decided in fp32: float64 may resolve a near-tie differently, which is not what is checked)."""
    sd, H = acoustic_sd64(), hp["hidden_size"]
    f64 = lambda k: u[k][None].double()
    lin = torch.nn.functional.linear
    tok, mel2ph = u["txt_tokens"][None], u["mel2ph"][None]
    with torch.no_grad():
        enc = O.fastspeech_encoder(tok, sd, hp) + O.note_encoder(u["note"][None], f64("note_dur"), u["note_type"][None], sd, H)
        spk = lin(f64("spk_embed"), sd["spk_embed_proj.weight"], sd["spk_embed_proj.bias"])[:, None]
        emo = lin(f64("emo_embed"), sd["emo_embed_proj.weight"], sd["emo_embed_proj.bias"])[:, None]
        _, logdur = O.duration_predictor((enc + spk + emo) * (tok > 0).double()[:, :, None], tok == 0, sd, hp)
        dec = O.expand_states(enc, mel2ph)
        style, _ = O.get_style(dec, f64("ref_mels"), u["ref_f0"].double(), sd, hp,
                               codes=torch.from_numpy(np.array(g["rq_codes"]))[None])
        pitch = O.f0_to_coarse(torch.from_numpy(np.array(g["f0_denorm"]))[None])
        tgt = (mel2ph > 0).double()[:, :, None]
        dinp = (dec + spk + torch.nn.functional.embedding(pitch, sd["pitch_embed.weight"], padding_idx=0) + emo + style) * tgt
        coarse = lin(O.fastspeech_decoder(dinp, sd, hp), sd["mel_out.weight"], sd["mel_out.bias"]) * tgt
    return {"style": style, "decoder_inp": dinp, "coarse_mel": coarse, "logdur": logdur}


def test_float64_oracle_matches_reference_fixtures():
    for name in ("ref_small_T4", "ref_padded_T4"):
        g, meta = golden(name)
        u = utt_from_meta(meta) if name == "ref_small_T4" else utt_from_fixture(g)
        r = _forward64(u, g, hp_for(meta["T"]))
        assert r["style"].dtype == torch.float64 and r["coarse_mel"].dtype == torch.float64
        errs = {k: _maxabs(r[k][0], g[k]) for k in ("style", "decoder_inp", "coarse_mel")}
        errs["logdur"] = _maxabs(r["logdur"][0], g["dur_logdur"])
        print(name, {k: f"{v:.2e}" for k, v in errs.items()})
        for k, e in errs.items():
            assert e < TOL, (name, k, e)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the oracle vs ref_registry
def _registry():
    g, meta = golden("ref_registry")
    d = registry_inputs(meta["seed"])
    assert np.array_equal(d["enc_tokens"].numpy(), g["in_enc_tokens"])
    assert np.array_equal(d["dec_x"][:, :2, :4].numpy(), g["in_dec_x_head"])
    return g, meta, d


def test_oracle_matches_reference_registry_modules_in_fp32_and_float64():
    g, meta, d = _registry()
    hp = hp_for(meta["T"])
    for sd, name in ((acoustic_sd(), "fp32"), (acoustic_sd64(), "float64")):
        with torch.no_grad():
            # the padded batches as the reference runs them (the oracle's masks follow the reference's)
            errs = {"encoder": _maxabs(O.fastspeech_encoder(d["enc_tokens"], sd, hp), g["enc_out"]),
                    "decoder": _maxabs(O.fastspeech_decoder(d["dec_x"].to(sd["decoder.pos_embed_alpha"].dtype), sd, hp),
                                       g["dec_out"])}
            for i in range(2):
                ref, f0 = d[f"style_ref_{i}"], d[f"style_f0_{i}"]
                dec = d[f"style_dec_{i}"]
                _, codes = O.get_style(dec, ref, f0, acoustic_sd(), hp)  # fp32 codes, as the reference decides them
                if name == "float64":
                    ref, f0, dec = ref.double(), f0.double(), dec.double()
                style, _ = O.get_style(dec, ref, f0, sd, hp, codes=codes if name == "float64" else None)
                errs[f"style_{i}"] = _maxabs(style[0], g[f"style_{i}"])
        print(name, {k: f"{v:.2e}" for k, v in errs.items()})
        for k, e in errs.items():
            assert e < TOL, (name, k, e)


def test_registry_fixture_padding_rows_and_b1_calls():
    """The reference's padded encoder / decoder batches: every padding row is exactly 0, and the longest utterance (no
    trailing padding; it holds the interior padding rows) equals its own B = 1 call.  Every utterance's B = 1 call on its
    rows up to the last non-padding row (what the facades hand the library) matches the oracle."""
    g, meta, d = _registry()
    hp = hp_for(meta["T"])
    tok, x = d["enc_tokens"], d["dec_x"]
    assert (g["enc_out"][tok.numpy() == 0] == 0).all()
    assert (g["dec_out"][x.abs().sum(-1).numpy() == 0] == 0).all()
    assert _maxabs(g["enc_out"][0], g["enc_b1_0"]) < TOL and _maxabs(g["dec_out"][0], g["dec_b1_0"]) < TOL
    el, dl = M._lengths_from_mask(tok != 0), M._true_lengths(x)
    assert el == [12, 7, 9] and dl == [24, 13, 19]
    with torch.no_grad():
        for b in range(3):
            for sd in (acoustic_sd(), acoustic_sd64()):
                e = O.fastspeech_encoder(tok[b:b + 1, :el[b]], sd, hp)[0]
                assert _maxabs(e, g[f"enc_b1_{b}"]) < TOL, b
                o = O.fastspeech_decoder(x[b:b + 1, :dl[b]].to(sd["decoder.pos_embed_alpha"].dtype), sd, hp)[0]
                assert _maxabs(o, g[f"dec_b1_{b}"]) < TOL, b


# ---------------------------------------------------------------------------------------------------------------------
# 3. facade host logic with a stand-in engine
class RecordingEngine:
    """Stands in for AcousticModel: records what each entry point receives and returns values the caller can trace back
    to the packed rows (the rows themselves, or a ramp)."""
    device = torch.device("cpu")

    def __init__(self):
        self.calls = {}

    def fft_encoder(self, tokens, offs):
        self.calls["fft_encoder"] = (tokens.clone(), np.array(offs))
        return tokens.float()[:, None].repeat(1, 256) + torch.arange(len(tokens), dtype=torch.float32)[:, None] * 1000

    def fft_decoder(self, x, offs):
        self.calls["fft_decoder"] = (x.clone(), np.array(offs))
        return x * 2 + 1

    def get_style(self, dec, fo, rm, rf, ro):
        self.calls["get_style"] = (dec.clone(), np.array(fo), rm.clone(), rf.clone(), np.array(ro))
        return dec + 1, None

    def denoiser_eval(self, which, x, uv, t, c, offs):
        self.calls["denoiser_eval"] = (which, x.clone(), None if uv is None else uv.clone(), t, c.clone(), np.array(offs))
        if which == 0:
            return x * 2
        return torch.stack([x, uv.float(), c[:, 0]], 1)


def test_fastspeech_encoder_facade_length_rule_and_layout():
    d = registry_inputs()
    eng = RecordingEngine()
    tok = torch.cat([d["enc_tokens"], torch.zeros(3, 2, dtype=torch.long)], 1)  # 2 more padding columns than any utterance
    out = M.FastspeechEncoder(eng)(tok)
    tight, offs = eng.calls["fft_encoder"]
    # the interior 0 token of utterance 0 stays in its sequence (the library masks it), its last real token is kept
    assert offs.tolist() == [0, 12, 19, 28]
    assert tight.dtype == torch.int32 and torch.equal(tight.long(), torch.cat([tok[0, :12], tok[1, :7], tok[2, :9]]))
    assert out.shape == (3, 14, 256)
    for b, (a, e) in enumerate(zip(offs[:-1], offs[1:])):
        n = e - a
        assert torch.equal(out[b, :n, 0], tok[b, :n].float() + torch.arange(a, e, dtype=torch.float32) * 1000)
        assert float(out[b, n:].abs().sum()) == 0.0


def test_fastspeech_decoder_facade_length_rule_and_layout():
    d = registry_inputs()
    eng = RecordingEngine()
    x = d["dec_x"]
    out = M.FastspeechDecoder(eng)(x)
    tight, offs = eng.calls["fft_decoder"]
    assert offs.tolist() == [0, 24, 37, 56]  # utterance 0's interior all-zero row 11 stays inside it
    assert torch.equal(tight, torch.cat([x[0, :24], x[1, :13], x[2, :19]]))
    assert out.shape == x.shape
    for b, n in enumerate((24, 13, 19)):
        assert torch.equal(out[b, :n], x[b, :n] * 2 + 1) and float(out[b, n:].abs().sum()) == 0.0


def test_get_style_facade_keeps_interior_zero_reference_rows():
    """A reference mel with an interior all-zero row (and one whose column 0 alone is 0) and trailing all-zero rows: the
    sequence handed to the library ends at the last non-zero row.  A count of the non-zero rows would keep the interior
    zero row and drop the last real one."""
    d = registry_inputs()
    eng = RecordingEngine()
    ref = torch.zeros(2, 34, 80)
    ref[0, :26] = d["style_ref_1"][0]  # interior all-zero row 9
    ref[1, :17] = d["style_ref_0"][0]
    ref[1, 4, 0] = 0
    f0 = torch.zeros(2, 34)
    f0[0, :26] = d["style_f0_1"]
    f0[1, :17] = d["style_f0_0"]
    dec = torch.zeros(2, 30, 256)
    dec[0] = d["style_dec_1"][0]
    dec[1, :21] = d["style_dec_0"][0]
    out = M.StyleSinger(engine=eng).get_style(dec, ref, {"ref_f0": f0}, infer=True)
    tdec, fo, rm, rf, ro = eng.calls["get_style"]
    assert fo.tolist() == [0, 30, 51] and ro.tolist() == [0, 26, 43]
    assert torch.equal(rm, torch.cat([ref[0, :26], ref[1, :17]])) and torch.equal(rf, torch.cat([f0[0, :26], f0[1, :17]]))
    assert float(rm[9].abs().sum()) == 0.0
    assert out.shape == (2, 30, 256) and torch.equal(out[1, :21], dec[1, :21] + 1) and float(out[1, 21:].abs().sum()) == 0
    # B = 1 with the reference's 1-D ref_f0
    M.StyleSinger(engine=eng).get_style(dec[:1], ref[:1, :26], {"ref_f0": f0[0, :26]}, infer=True)
    assert eng.calls["get_style"][4].tolist() == [0, 26]


def test_diffnet_facade_layout():
    """DiffNet: spec [B,1,M,F] and cond [B,H,F] go to the library as frame rows [B*F, M] / [B*F, H]; the result comes back
    as [B,1,M,F]."""
    g = torch.Generator().manual_seed(3)
    B, Mb, Fr, H = 3, 80, 7, 256
    spec, cond = torch.randn(B, 1, Mb, Fr, generator=g), torch.randn(B, H, Fr, generator=g)
    eng = RecordingEngine()
    out = M.DiffNet(eng)(spec, torch.tensor([5, 5, 5]), cond)
    which, x, uv, t, c, offs = eng.calls["denoiser_eval"]
    assert which == 0 and uv is None and t == 5 and offs.tolist() == [0, 7, 14, 21]
    for b in range(B):
        for f in range(Fr):
            assert torch.equal(x[b * Fr + f], spec[b, 0, :, f]) and torch.equal(c[b * Fr + f], cond[b, :, f])
    assert out.shape == spec.shape and out.is_contiguous() and torch.equal(out, spec * 2)


def test_ddiffnet_facade_layout():
    """DDiffNet: f0 [B,1,F], uv [B,F] and cond [B,H,F] as frame rows; [B*F, 3] back as [B,3,F], times nonpadding."""
    g = torch.Generator().manual_seed(4)
    B, Fr, H = 2, 9, 256
    f0, cond = torch.randn(B, 1, Fr, generator=g), torch.randn(B, H, Fr, generator=g)
    uv = (torch.rand(B, Fr, generator=g) < 0.5).long()
    eng = RecordingEngine()
    for which in (1, 2):
        out = M.DDiffNet(eng, which)(f0, uv, torch.tensor([2, 2]), cond)
        w, x, u, t, c, offs = eng.calls["denoiser_eval"]
        assert w == which and t == 2 and offs.tolist() == [0, 9, 18] and u.dtype == torch.int32
        assert torch.equal(x, f0.reshape(-1)) and torch.equal(u.long(), uv.reshape(-1))
        assert out.shape == (B, 3, Fr)
        assert torch.equal(out[:, 0], f0[:, 0]) and torch.equal(out[:, 1], uv.float()) and torch.equal(out[:, 2], cond[:, 0])
    nonpad = torch.ones(B, Fr)
    nonpad[1, 6:] = 0
    out = M.DDiffNet(eng, 1)(f0, uv, torch.tensor([2, 2]), cond, nonpad)
    assert float(out[1, :, 6:].abs().sum()) == 0.0 and torch.equal(out[0, 0], f0[0, 0])
