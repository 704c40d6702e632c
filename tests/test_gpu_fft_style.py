"""The deterministic half of the acoustic model through its own entry points, against the float64 oracle: ssb_fft_encoder,
ssb_fft_decoder, ssb_get_style and ssb_predict_durations on B > 1, the facades built on them, and the workspace contract
of the three drop-ins.

Each entry point runs at three sizes so that every kernel path is covered: a small batch (< 8 row tiles: FFMA GEMMs and
fp32 attention), a mid batch (44 row tiles: QKV, FFN1 and aligner linear1 on the CTA-pair kernel, the 256-wide GEMMs on
tc<64>) and the bench's batch64 utterances (every decoder and aligner GEMM on the CTA-pair kernel).  Every call asserts
the tensor-core GEMM variants it launched, so that a change of threshold cannot move a test off the path it covers.

The float64 oracle is oracle/stylesinger_oracle.py on the state dict cast to float64 (tests/test_registry_cpu.py pins it
to the reference); get_style's float64 run takes the RVQ codes of the fp32 oracle, which the kernel must match exactly.
Errors are max |a - b| / max(1, |b|) per element.  The bars were set from errors measured on an H100 SXM (80 GB) at no
more than 4x the largest measured error; each test prints what it measured.
"""
import ctypes as C
import time

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from tests.common import acoustic_engine, acoustic_sd, acoustic_sd64, golden, hp_for, registry_inputs
from tests.gpu_checks import variant

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T = 4
HP = hp_for(T)

# bars per batch size, each at most 4x the largest error measured on an H100 80GB HBM3 (SXM, 700 W power limit); the
# measured values are in the comments.  0 means bit-identical (the small batch runs the per-utterance FFMA path).
EXACT = float(np.nextafter(0, 1))
BARS = {
    "small": {"enc_oracle": 7e-6,            # 1.7e-6
              "dec_oracle": 8e-6,            # 1.9e-6
              "dec_paths": EXACT, "dec_solo": EXACT,
              "style_oracle": 1.4e-5,        # 3.5e-6
              "style_solo": EXACT},
    "mid": {"enc_oracle": 1.1e-5,            # 2.9e-6
            "dec_oracle": 1.6e-4,            # 4.1e-5
            "dec_paths": 1.6e-4,             # 4.2e-5 tensor cores vs FFMA
            "dec_solo": 6e-5,                # 1.6e-5
            "style_oracle": 1.5e-4,          # 3.8e-5
            "style_solo": 1.3e-4},           # 3.3e-5
    "bench": {"enc_oracle": 1e-5,            # 2.6e-6
              "enc_fwd_oracle": 1e-5,        # 2.7e-6
              "dec_oracle": 2e-4,            # 5.2e-5
              "dec_paths": 2e-4,             # 5.2e-5
              "dec_solo": 8e-5,              # 2.2e-5
              "chain": 1e-5,                 # 2.7e-6
              "style_oracle": 1e-4,          # 2.6e-5
              "style_solo": 8e-5},           # 2.2e-5
    "durations": {"logdur_oracle": 4e-7},    # 1.1e-7
    "facades": {"facade": 1.4e-5,            # 3.5e-6 vs the float64 oracle
                "facade_ref": 1.6e-5,        # 4.0e-6 vs the reference fixtures
                "facade_dn": 1.6e-5},        # 4.2e-6 denoisers vs the fp32 oracle
}

SMALL = [1, 2, 63, 64, 65, 127, 128]                             # 7 row tiles
MID = [129, 1, 2, 63, 64, 65, 127, 128, 1200, 1300, 1700]        # 44 row tiles
SMALL_REF = [64, 1, 65, 1125, 1, 64, 65]                         # frames shorter and longer than the reference
MID_REF = [1125, 64, 65, 1, 1125, 1, 64, 65, 1125, 200, 1125]
HALF = 1e-4  # a predicted duration may round the other way when exp(logdur) - 1 is this close to a half-integer


def _offs(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


def _ntiles(lens):
    return sum((int(n) + 127) // 128 for n in lens)


def _rel(a, b):
    a = a.detach().cpu().double() if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a, np.float64))
    b = b.detach().cpu().double() if isinstance(b, torch.Tensor) else torch.as_tensor(np.asarray(b, np.float64))
    if a.numel() == 0:
        return 0.0
    return float(((a - b).abs() / b.abs().clamp(min=1.0)).max())


def _report(name, errs, bars):
    for k, e in errs.items():
        print(f"{name}: {k} {e:.3e} (bar {bars[k]:.1e})")
    bad = {k: e for k, e in errs.items() if not e < bars[k]}
    assert not bad, (name, bad)


# ---------------------------------------------------------------------------------------------------------------------
# which tensor-core GEMM variants a call must launch (conv_gemm_tc's dispatch, tests/gpu_checks.py; none of these GEMMs is a
# 3-tap conv, so none takes the tap-reuse kernel); the FFMA path (< 8 row tiles) launches none
def _expect(gemms):
    out = {}
    for nt, N in gemms:
        k = variant(nt, N, "GENERIC", 1)
        out[k] = out.get(k, 0) + 1
    return out


def expected_decoder(lens):
    nt = _ntiles(lens)
    if nt < 8:
        return {}
    return _expect([(nt, 768), (nt, 256), (nt, 1024), (nt, 256)] * HP["dec_layers"])


def expected_style(flens, rlens):
    nt, ntr = _ntiles(flens), _ntiles(rlens)
    if nt < 8:
        return {}
    return _expect([(nt, 256), (ntr, 512), (nt, 256), (nt, 2048), (nt, 256)] * 2)


def _launched(fn):
    from stylesinger_b200._lib import variant_launches
    torch.cuda.synchronize()
    before = variant_launches()
    r = fn()
    torch.cuda.synchronize()
    after = variant_launches()
    return r, {k: after[k] - before.get(k, 0) for k in after if after[k] > before.get(k, 0)}


def _check_variants(tag, got, want):
    print(f"{tag}: tensor-core GEMM variants launched {got}")
    assert got == want, (tag, got, want)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
def _tokens(lens, seed):
    """Token sequences with trailing padding tokens (0) in some utterances and one interior 0 token."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, n in enumerate(lens):
        t = torch.randint(3, synth.N_TOKENS, (n,), generator=g)
        if n >= 60 and i % 3 == 0:
            t[-4:] = 0
        if n >= 60 and i % 3 == 1:
            t[n // 2] = 0
        if n == 128:
            t[-1] = 0
        out.append(t)
    return out


def _frames(lens, seed):
    """Decoder inputs with interior and trailing all-zero frames and rows whose column 0 alone is 0."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for n in lens:
        x = torch.randn(n, 256, generator=g)
        if n >= 60:
            x[n // 6: n // 6 + max(1, n // 20)] = 0
            x[n - max(1, n // 25):] = 0
            x[n // 3, 0] = 0
        out.append(x)
    return out


def _refs(lens, seed):
    """Reference mels (synth.make_utterance's distribution) with trailing all-zero rows and a column-0-only zero row."""
    out = []
    for i, R in enumerate(lens):
        u = synth.make_utterance(1.0, utt_idx=300 + seed + i, ref_frames=R, frames=8, phones=4)
        ref, f0 = u["ref_mels"], u["ref_f0"]
        if R >= 64:
            ref[R // 2, 0] = 0
            ref[R - R // 16:] = 0
            f0[R - R // 16:] = 0
        out.append((ref, f0))
    return out


def _cat_dev(xs, dtype=torch.float32):
    return torch.cat(xs).to(DEV, dtype).contiguous()


def _split(x, offs):
    x = x.cpu()
    return [x[int(offs[i]):int(offs[i + 1])] for i in range(len(offs) - 1)]


# ---------------------------------------------------------------------------------------------------------------------
# float64 oracle (memoised per input)
_OR = {}


def _or_encoder(key, tok):
    if key not in _OR:
        with torch.no_grad():
            _OR[key] = O.fastspeech_encoder(tok[None], acoustic_sd64(), HP)[0]
    return _OR[key]


def _or_decoder(key, x):
    if key not in _OR:
        with torch.no_grad():
            _OR[key] = O.fastspeech_decoder(x.double()[None], acoustic_sd64(), HP)[0]
    return _OR[key]


def _or_style(key, dec, ref, f0):
    """(float64 style with the fp32 codes, fp32 codes)."""
    if key not in _OR:
        with torch.no_grad():
            _, codes = O.local_style_adaptor(ref[None], f0, acoustic_sd(), HP)
            st, _ = O.get_style(dec.double()[None], ref.double()[None], f0.double(), acoustic_sd64(), HP, codes=codes)
        _OR[key] = (st[0], codes[0])
    return _OR[key]


# ---------------------------------------------------------------------------------------------------------------------
# the bench batch: the utterances of make_workload("batch64") at one GPU (seed 1234, 1,125-frame references), every
# eighth with padding frames, through the forward
_BENCH = {}


def bench_batch():
    if not _BENCH:
        from stylesinger_b200.engine import pack_batch
        secs = synth.batch_seconds(64, seed=1234)
        utts = [synth.make_utterance(float(s), utt_idx=i) for i, s in enumerate(secs)]
        for u in utts[::8]:  # padding frames (an interior and a trailing run), so the decoder's row masks matter at scale
            n = len(u["mel2ph"])
            u["mel2ph"][n // 3: n // 3 + 100] = 0
            u["mel2ph"][n - 30:] = 0
        pb = pack_batch(utts).to(DEV)
        assert pb.total_frames == 110119 and int(pb.ph_offsets[-1]) == 4405
        m = acoustic_engine(T)
        out = m.forward(pb, seed=1, skip_mel_diffusion=True, want=("encoder_out", "decoder_inp", "coarse_mel", "mel2ph"))
        _BENCH.update(utts=utts, pb=pb, out={k: v.clone() for k, v in out.items()})
    return _BENCH


# ---------------------------------------------------------------------------------------------------------------------
# ssb_fft_encoder
@pytest.mark.parametrize("size", ["small", "mid", "bench"])
def test_fft_encoder_matches_float64_and_solo(size):
    m = acoustic_engine(T)
    if size == "bench":
        b = bench_batch()
        toks = [u["txt_tokens"] for u in b["utts"]]
    else:
        toks = _tokens(SMALL if size == "small" else MID, 11)
    offs = _offs([len(t) for t in toks])
    out, launched = _launched(lambda: m.fft_encoder(_cat_dev(toks, torch.int32), offs))
    _check_variants(f"encoder {size}", launched, {})  # always the FFMA path
    errs = {"enc_oracle": 0.0}
    for i, (t, y) in enumerate(zip(toks, _split(out, offs))):
        pad = t == 0
        assert float(y[pad].abs().max()) == 0.0 if pad.any() else True, i
        errs["enc_oracle"] = max(errs["enc_oracle"], _rel(y, _or_encoder(("enc", size, i), t)))
        if size != "bench" or i % 8 == 0:
            solo = m.fft_encoder(t.to(DEV, torch.int32).contiguous(), _offs([len(t)])).cpu()
            assert torch.equal(solo, y), (size, i)
    if size == "bench":  # the forward's encoder_out adds the note encoder to the same encoder
        sd = acoustic_sd64()
        po = b["pb"].ph_offsets
        eo = _split(b["out"]["encoder_out"], po)
        e = 0.0
        with torch.no_grad():
            for i, u in enumerate(b["utts"]):
                ref = _or_encoder(("enc", size, i), u["txt_tokens"]) + O.note_encoder(
                    u["note"][None], u["note_dur"][None].double(), u["note_type"][None], sd, 256)[0]
                e = max(e, _rel(eo[i], ref))
        errs["enc_fwd_oracle"] = e
    _report(f"ssb_fft_encoder {size} ({len(toks)} utterances, {int(offs[-1])} phones)", errs, BARS[size])


# ---------------------------------------------------------------------------------------------------------------------
# ssb_fft_decoder
def _decoder_inputs(size):
    if size == "bench":
        b = bench_batch()
        return _split(b["out"]["decoder_inp"], b["pb"].frame_offsets)
    return _frames(SMALL if size == "small" else MID, 21)


def _fft_decoder_both_paths(m, xs, offs):
    from stylesinger_b200._lib import lib
    x = _cat_dev(xs)
    on, launched = _launched(lambda: m.fft_decoder(x, offs).clone())
    try:
        m.set_fft_tensor_cores(False)
        lib.ssb_set_attention_tensor_cores(0)
        off, launched_off = _launched(lambda: m.fft_decoder(x, offs).clone())
    finally:
        m.set_fft_tensor_cores(True)
        lib.ssb_set_attention_tensor_cores(1)
    assert launched_off == {}
    return on, off, launched


@pytest.mark.parametrize("size", ["small", "mid", "bench"])
def test_fft_decoder_matches_float64_other_path_and_solo(size):
    m = acoustic_engine(T)
    xs = _decoder_inputs(size)
    lens = [len(x) for x in xs]
    offs = _offs(lens)
    on, off, launched = _fft_decoder_both_paths(m, xs, offs)
    want = expected_decoder(lens)
    if size == "bench":
        assert want == {"tc2<64,GENERIC>": 16}, want
    if size == "mid":
        assert want.get("tc2<64,GENERIC>") == 8 and want.get("tc<64,GENERIC>") == 8, want
    _check_variants(f"decoder {size}", launched, want)
    errs = {"dec_oracle": 0.0, "dec_paths": _rel(on, off), "dec_solo": 0.0}
    t0 = time.time()
    for i, (x, y) in enumerate(zip(xs, _split(on, offs))):
        keep = x.abs().sum(-1) > 0
        assert float(y[~keep].abs().max()) == 0.0 if (~keep).any() else True, i
        errs["dec_oracle"] = max(errs["dec_oracle"], _rel(y, _or_decoder(("dec", size, i), x)))
        solo = m.fft_decoder(x.to(DEV).contiguous(), _offs([len(x)])).cpu()
        errs["dec_solo"] = max(errs["dec_solo"], _rel(y, solo))
    print(f"decoder {size}: oracle and solo checks of {len(xs)} utterances took {time.time() - t0:.1f} s")
    if size == "bench":
        # chain: mel_out on the host, times the padding-frame mask (stylesinger_oracle.py: coarse = mel_out(dec) * tgt)
        b = bench_batch()
        sd = acoustic_sd()
        keep = (b["out"]["mel2ph"].cpu() > 0).double()[:, None]
        coarse = (on.cpu().double() @ sd["mel_out.weight"].double().t() + sd["mel_out.bias"].double()) * keep
        errs["chain"] = _rel(b["out"]["coarse_mel"], coarse)
    _report(f"ssb_fft_decoder {size} ({len(xs)} utterances, {int(offs[-1])} frames, {_ntiles(lens)} row tiles)", errs,
            BARS[size])


# ---------------------------------------------------------------------------------------------------------------------
# ssb_get_style
def _style_inputs(size):
    if size == "bench":
        b = bench_batch()
        decs = _split(b["out"]["decoder_inp"], b["pb"].frame_offsets)
        refs = [(u["ref_mels"], u["ref_f0"]) for u in b["utts"]]
        return decs, refs
    fl, rl = (SMALL, SMALL_REF) if size == "small" else (MID, MID_REF)
    g = torch.Generator().manual_seed(31)
    return [torch.randn(n, 256, generator=g) for n in fl], _refs(rl, 1 if size == "small" else 2)


@pytest.mark.parametrize("size", ["small", "mid", "bench"])
def test_get_style_codes_exact_and_style_matches_float64(size):
    m = acoustic_engine(T)
    decs, refs = _style_inputs(size)
    fl, rl = [len(d) for d in decs], [len(r) for r, _ in refs]
    fo, ro = _offs(fl), _offs(rl)
    (style, codes), launched = _launched(lambda: m.get_style(_cat_dev(decs), fo, _cat_dev([r for r, _ in refs]),
                                                             _cat_dev([f for _, f in refs]), ro))
    want = expected_style(fl, rl)
    if size == "bench":
        assert want == {"tc2<64,GENERIC>": 10}, want
    _check_variants(f"get_style {size}", launched, want)
    assert codes.shape == (int(ro[-1]), HP["rq_depth"])
    errs = {"style_oracle": 0.0, "style_solo": 0.0}
    t0 = time.time()
    for i, (d, (r, f), s, c) in enumerate(zip(decs, refs, _split(style, fo), _split(codes, ro))):
        st64, c32 = _or_style(("style", size, i), d, r, f)
        assert torch.equal(c.long(), c32), (size, i, int((c.long() != c32).sum()))
        errs["style_oracle"] = max(errs["style_oracle"], _rel(s, st64))
        if size != "bench" or i % 8 == 0:
            s1, c1 = m.get_style(d.to(DEV).contiguous(), _offs([len(d)]), r.to(DEV).contiguous(), f.to(DEV).contiguous(),
                                 _offs([len(r)]))
            assert torch.equal(c1.cpu(), c), (size, i)
            errs["style_solo"] = max(errs["style_solo"], _rel(s, s1))
    print(f"get_style {size}: oracle checks of {len(decs)} utterances took {time.time() - t0:.1f} s")
    _report(f"ssb_get_style {size} ({len(decs)} utterances, {int(fo[-1])} frames, {int(ro[-1])} reference rows)", errs,
            BARS[size])


def test_get_style_codes_out_column_layout():
    """codes_out is [sum R, depth] row-major: column d of utterance b's rows holds depth d's index (ssb_rvq_lookup writes
    the same layout); the columns are distinct sequences, so a column written one place off cannot pass."""
    m = acoustic_engine(T)
    decs, refs = _style_inputs("small")
    ro = _offs([len(r) for r, _ in refs])
    _, codes = m.get_style(_cat_dev(decs), _offs([len(d) for d in decs]), _cat_dev([r for r, _ in refs]),
                           _cat_dev([f for _, f in refs]), ro)
    with torch.no_grad():
        per = [O.local_style_adaptor(r[None], f, acoustic_sd(), HP) for r, f in refs]
    ref = torch.cat([c[0] for _, c in per])
    codes = codes.cpu().long()
    assert codes.shape == ref.shape == (int(ro[-1]), 4)
    for d in range(4):
        assert torch.equal(codes[:, d], ref[:, d]), d
    assert all(not torch.equal(ref[:, d], ref[:, d + 1]) for d in range(3))


# ---------------------------------------------------------------------------------------------------------------------
# ssb_predict_durations on B > 1, and the length regulator behind forward(dur=...)
def _dur_batch():
    b = bench_batch()
    extra = []
    for i, (s, pad) in enumerate(((0.5, 3), (1.2, 5), (0.3, 1))):
        u = synth.make_utterance(s, utt_idx=200 + i)
        for k in ("txt_tokens", "note", "note_type", "note_dur"):
            u[k] = torch.cat([u[k], torch.zeros(pad, dtype=u[k].dtype)])
        extra.append(u)
    return b["utts"][:20] + extra[:2] + b["utts"][20:] + extra[2:]


def test_predict_durations_batched_matches_oracle_and_length_regulator():
    from stylesinger_b200.engine import pack_batch
    m = acoustic_engine(T)
    utts = _dur_batch()
    pb = pack_batch(utts, use_mel2ph=False).to(DEV)
    dur, logdur = m.predict_durations(pb)
    dur, logdur = dur.cpu(), logdur.cpu()
    po = pb.ph_offsets
    sd, sd64 = acoustic_sd(), acoustic_sd64()
    lin = torch.nn.functional.linear
    e_log, near, dur_or = 0.0, [], []
    with torch.no_grad():
        for i, u in enumerate(utts):
            tok = u["txt_tokens"][None]
            outs = {}
            for name, s in (("fp32", sd), ("f64", sd64)):
                cast = (lambda t: t.double()) if name == "f64" else (lambda t: t.float())
                enc = O.fastspeech_encoder(tok, s, HP) + O.note_encoder(u["note"][None], cast(u["note_dur"][None]),
                                                                        u["note_type"][None], s, 256)
                spk = lin(cast(u["spk_embed"][None]), s["spk_embed_proj.weight"], s["spk_embed_proj.bias"])[:, None]
                emo = lin(cast(u["emo_embed"][None]), s["emo_embed_proj.weight"], s["emo_embed_proj.bias"])[:, None]
                outs[name] = O.duration_predictor((enc + spk + emo) * cast((tok > 0).float())[:, :, None], tok == 0, s, HP)
            a, e = int(po[i]), int(po[i + 1])
            ld64 = outs["f64"][1][0, :, 0]
            e_log = max(e_log, _rel(logdur[a:e], ld64))
            d32 = outs["fp32"][0][0].int()
            dur_or.append(d32)
            frac = (ld64.exp() - 1) - torch.floor(ld64.exp() - 1)
            close = ((frac - 0.5).abs() < HALF * ld64.exp().clamp(min=1)).numpy()
            for j in np.nonzero((dur[a:e] != d32).numpy())[0]:
                assert close[j], (i, j, int(dur[a + j]), int(d32[j]), float(ld64[j]))
                near.append((i, int(j)))
            assert (dur[a:e][tok[0] == 0] == 0).all()
    print(f"durations: {int(po[-1])} phones in {len(utts)} utterances, {len(near)} differ from the fp32 oracle, all "
          f"within the bar of a half-integer: {near}")
    _report("ssb_predict_durations", {"logdur_oracle": e_log}, BARS["durations"])
    # forward(dur=...) regulates the durations per utterance: mel2ph equals the oracle's length_regulator on them
    lens = [int(dur[po[i]:po[i + 1]].sum()) for i in range(len(utts))]
    pb.frame_offsets = _offs(lens)
    out = m.forward(pb, seed=3, skip_mel_diffusion=True, dur=dur.to(DEV).contiguous(), want=("mel2ph",))
    m2p = _split(out["mel2ph"], pb.frame_offsets)
    for i, u in enumerate(utts):
        d = dur[po[i]:po[i + 1]].long()[None]
        ref = O.length_regulator(d, u["txt_tokens"][None] == 0)[0]
        assert torch.equal(m2p[i].long(), ref), i


# ---------------------------------------------------------------------------------------------------------------------
# the facades on the real engine
def test_facades_match_reference_registry_fixture_and_oracle():
    from stylesinger_b200 import modules as M
    m = acoustic_engine(T)
    g, meta = golden("ref_registry")
    d = registry_inputs(meta["seed"])
    errs = {"facade": 0.0, "facade_ref": 0.0, "facade_dn": 0.0}
    enc = M.FastspeechEncoder(m)(d["enc_tokens"]).cpu()
    dec = M.FastspeechDecoder(m)(d["dec_x"]).cpu()
    assert enc.shape == (3, 12, 256) and dec.shape == (3, 24, 256)
    for b, (ne, nd) in enumerate(zip((12, 7, 9), (24, 13, 19))):
        errs["facade_ref"] = max(errs["facade_ref"], _rel(enc[b, :ne], g[f"enc_b1_{b}"]), _rel(dec[b, :nd], g[f"dec_b1_{b}"]))
        errs["facade"] = max(errs["facade"], _rel(enc[b, :ne], _or_encoder(("reg_enc", b), d["enc_tokens"][b, :ne])),
                             _rel(dec[b, :nd], _or_decoder(("reg_dec", b), d["dec_x"][b, :nd])))
        assert float(enc[b, ne:].abs().sum()) == 0 and float(dec[b, nd:].abs().sum()) == 0
    assert float(enc[0, 3].abs().sum()) == 0 and float(dec[0, 11].abs().sum()) == 0  # interior padding rows
    errs["facade_ref"] = max(errs["facade_ref"], _rel(enc[0], g["enc_out"][0]), _rel(dec[0], g["dec_out"][0]))
    ss = M.StyleSinger(engine=m)
    for i in range(2):  # B = 1; reference mel 1 holds an interior all-zero row
        st = ss.get_style(d[f"style_dec_{i}"], d[f"style_ref_{i}"], {"ref_f0": d[f"style_f0_{i}"]}, infer=True).cpu()
        errs["facade_ref"] = max(errs["facade_ref"], _rel(st[0], g[f"style_{i}"]))
        st64, _ = _or_style(("reg_style", i), d[f"style_dec_{i}"][0], d[f"style_ref_{i}"][0], d[f"style_f0_{i}"])
        errs["facade"] = max(errs["facade"], _rel(st[0], st64))
    # a padded get_style batch: each utterance as at B = 1 on its rows up to its last non-zero reference row
    decs, refs = _style_inputs("small")
    Fm, Rm = max(len(x) for x in decs), max(len(r) for r, _ in refs)
    pd, pr, pf = torch.zeros(len(decs), Fm, 256), torch.zeros(len(decs), Rm + 3, 80), torch.zeros(len(decs), Rm + 3)
    for b, (x, (r, f)) in enumerate(zip(decs, refs)):
        pd[b, :len(x)], pr[b, :len(r)], pf[b, :len(r)] = x, r, f
    st = ss.get_style(pd, pr, {"ref_f0": pf}, infer=True).cpu()
    for b, (x, (r, f)) in enumerate(zip(decs, refs)):
        nr = int((r.abs().sum(-1) > 0).nonzero()[-1]) + 1
        st64, _ = _or_style(("pad_style", b), x, r[:nr], f[:nr])
        errs["facade"] = max(errs["facade"], _rel(st[b, :len(x)], st64))
    # the denoisers: the reference's own single evaluations (ref_small_T4) and an oracle batch of three
    gs, ms = golden("ref_small_T4")
    assert ms["T"] == T
    cond = torch.from_numpy(gs["dn_cond"])[None]
    e1 = M.DiffNet(m)(torch.from_numpy(gs["dn_spec"])[None, None], torch.tensor([T - 1]), cond).cpu()
    f0 = torch.from_numpy(gs["dd_f0"])[None, None]
    uv = torch.from_numpy(gs["dd_uv"])[None]
    e2 = M.DDiffNet(m, 1)(f0, uv, torch.tensor([1]), cond, torch.ones(1, f0.shape[-1])).cpu()
    e3 = M.DDiffNet(m, 2)(f0, uv, torch.tensor([0]), cond).cpu()
    errs["facade_ref"] = max(errs["facade_ref"], _rel(e1[0, 0], gs["dn_out"]), _rel(e2[0], gs["dd_out"]),
                             _rel(e3[0], gs["dd_out_inp"]))
    gg = torch.Generator().manual_seed(41)
    spec, cnd = torch.randn(3, 1, 80, 70, generator=gg), torch.randn(3, 256, 70, generator=gg)
    f0b, uvb = torch.randn(3, 1, 70, generator=gg), (torch.rand(3, 70, generator=gg) < 0.4).long()
    with torch.no_grad():  # the fp32 oracle: its diffusion-step embedding is fp32 like the reference's
        r1 = O.diffnet(spec, torch.tensor([2, 2, 2]), cnd, acoustic_sd(), HP)
        r2 = O.ddiffnet(f0b, uvb, torch.tensor([3, 3, 3]), cnd, acoustic_sd(), HP, "gm_diffnet_inpainte.")
    errs["facade_dn"] = max(_rel(M.DiffNet(m)(spec, torch.tensor([2, 2, 2]), cnd), r1),
                            _rel(M.DDiffNet(m, 2)(f0b, uvb, torch.tensor([3, 3, 3]), cnd), r2))
    _report("facades", errs, BARS["facades"])


# ---------------------------------------------------------------------------------------------------------------------
# workspace contract of the three drop-ins
TAIL = 1 << 20


def _raw(m, which, size, ws, nbytes):
    from stylesinger_b200._lib import check, lib
    p = lambda t: C.c_void_p(t.data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if which == "encoder":
        toks = _tokens(SMALL if size == "small" else MID, 11)
        offs = _offs([len(t) for t in toks])
        x = _cat_dev(toks, torch.int32)
        out = torch.empty(int(offs[-1]), 256, device=DEV)
        check(lib.ssb_fft_encoder(m._h, p(x), offs.ctypes.data, len(toks), p(out), p(ws), nbytes, stream))
        outs = (out,)
    elif which == "decoder":
        xs = _decoder_inputs(size)
        offs = _offs([len(x) for x in xs])
        x = _cat_dev(xs)
        out = torch.empty(int(offs[-1]), 256, device=DEV)
        check(lib.ssb_fft_decoder(m._h, p(x), offs.ctypes.data, len(xs), p(out), p(ws), nbytes, stream))
        outs = (out,)
    else:
        decs, refs = _style_inputs(size)
        fo, ro = _offs([len(d) for d in decs]), _offs([len(r) for r, _ in refs])
        style = torch.empty(int(fo[-1]), 256, device=DEV)
        codes = torch.empty(int(ro[-1]), 4, dtype=torch.int32, device=DEV)
        check(lib.ssb_get_style(m._h, p(_cat_dev(decs)), fo.ctypes.data, p(_cat_dev([r for r, _ in refs])),
                                p(_cat_dev([f for _, f in refs])), ro.ctypes.data, len(decs), p(style), p(codes), p(ws),
                                nbytes, stream))
        outs = (style, codes)
    torch.cuda.synchronize()
    return outs


def _ws_bytes(m, which, size):
    from stylesinger_b200._lib import lib
    if which == "encoder":
        offs = _offs([len(t) for t in _tokens(SMALL if size == "small" else MID, 11)])
        n = lib.ssb_fft_workspace_bytes(m._h, 0, offs.ctypes.data, len(offs) - 1)
    elif which == "decoder":
        offs = _offs(SMALL if size == "small" else MID)
        n = lib.ssb_fft_workspace_bytes(m._h, 1, offs.ctypes.data, len(offs) - 1)
    else:
        fl, rl = (SMALL, SMALL_REF) if size == "small" else (MID, MID_REF)
        fo, ro = _offs(fl), _offs(rl)
        n = lib.ssb_get_style_workspace_bytes(m._h, fo.ctypes.data, ro.ctypes.data, len(fl))
    assert n > 0
    return int(n)


@pytest.mark.parametrize("which", ["encoder", "decoder", "get_style"])
def test_workspace_contract(which):
    """The queried size is enough, the call never reads workspace bytes it has not written (0xFF-filled and zeroed
    workspaces give the same bits) and never writes past the queried size (a 1 MB sentinel tail survives)."""
    m = acoustic_engine(T)
    g = torch.Generator(device=DEV).manual_seed(7)
    sentinel = torch.randint(0, 256, (TAIL,), generator=g, device=DEV, dtype=torch.int32).to(torch.uint8)
    for size in ("small", "mid"):
        n = _ws_bytes(m, which, size)
        ws = torch.empty(n + TAIL, dtype=torch.uint8, device=DEV)
        ws[n:] = sentinel
        ws[:n].fill_(0xFF)
        a = [t.clone() for t in _raw(m, which, size, ws, n)]
        assert torch.equal(ws[n:], sentinel), (which, size, "wrote past the queried workspace size")
        ws[:n].zero_()
        b = _raw(m, which, size, ws, n)
        assert torch.equal(ws[n:], sentinel), (which, size)
        for x, y in zip(a, b):
            assert (not x.is_floating_point() or torch.isfinite(x).all()) and torch.equal(x, y), (which, size)
        print(f"workspace {which} {size}: {n} bytes, bit-identical on 0xFF / zeroed workspaces, sentinel tail intact")
        del ws
