"""The FastSpeech 2 mel decoder (decoder: fft) and speaker ids (use_spk_id) on the CUDA path: every configuration of
tests/golden/ref_fft_spkid.npz against the unmodified reference on FFMA and on tensor cores, ragged batches at bench
lengths against the test oracle, the FFT model against the DiffSinger model's coarse mel, the speaker table against the
Linear projection it replaces, the documented errors (with no kernel launched), the workspace dry run, keyed seeds and
padding frames."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from tests.common import engine_noise_from_stream, fft_spkid_hp, fft_spkid_sd, golden, utt_from_meta

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_C = {}
CONFIGS = ("fft_gmdiff", "fft_conv", "spkid_diffsinger", "spkid_fft", "fft_no_emo_style")


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    """Free the cached models and their workspaces when the module ends (the modules after it keep the device memory)."""
    yield
    _C.clear()
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _maxabs(a, b):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def _fixture():
    if "g" not in _C:
        _C["g"], _C["meta"] = golden("ref_fft_spkid")
    return _C["g"], _C["meta"]


def _cfg(c, T=None):
    _, meta = _fixture()
    return {"T": T or meta["T"], "overrides": meta["configs"][c]["overrides"]}


def _model(c, T=None):
    from stylesinger_b200.engine import AcousticModel
    key = (c, T)
    if key not in _C:
        _C[key] = AcousticModel(fft_spkid_sd(_cfg(c, T)), fft_spkid_hp(_cfg(c, T)), DEV)
    m = _C[key]
    m.set_tensor_cores(True)
    m.set_persistent(True)
    return m


def _noise(hp, seed, Fr):
    """The forward's draws from NoiseSource(seed) in the C ABI's layout: the two F0 samplers' (gmdiff), then the mel
    sampler's T + 1 (a DiffSinger model only: an FFT model draws no mel noise).  None when nothing is drawn."""
    T = hp["timesteps"]
    if hp["f0_gen"] == "conv":
        if hp["decoder"] == "fft":
            return None
        ns = O.NoiseSource(seed)
        return {"mel": torch.stack([ns.randn((1, 1, 80, Fr))[0, 0].t() for _ in range(T + 1)]).contiguous().to(DEV)}
    n = engine_noise_from_stream(seed, T, T, Fr, DEV)[0]
    if hp["decoder"] == "fft":
        del n["mel"]
    return n


def _f0_noise(per_utt):
    """Per-utterance injected F0 noise concatenated along the frame axis (an FFT model takes no mel noise)."""
    return {k: [torch.cat([n[k][i] for n in per_utt], dim=1).contiguous() for i in range(2)] for k in ("f0_gauss", "f0_unif")}


def _want(hp):
    w = ["mel_out", "f0_denorm", "pitch_pred", "decoder_inp", "mel2ph", "spk_proj"]
    w += ["emo_proj"] if hp["emo"] else []
    w += ["style", "rq_codes"] if hp["style"] else []
    return tuple(w)


def _utt(meta):
    u = utt_from_meta(meta)
    u["spk_id"] = meta["spk_id"]
    return u


def _forward(m, u, seed, use_mel2ph=True):
    pb = m.pack_batch([u], use_mel2ph=use_mel2ph).to(DEV)
    dur = None
    if not use_mel2ph:
        dur, _ = m.predict_durations(pb)
        pb.frame_offsets = np.array([0, int(dur.sum())], np.int32)
    out = m.forward(pb, noise=_noise(m.hp, seed, int(pb.frame_offsets[-1])), dur=dur, want=_want(m.hp))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("tc", [False, True], ids=["ffma", "tc"])
@pytest.mark.parametrize("c", CONFIGS)
def test_forward_matches_reference_golden(c, tc):
    g, meta = _fixture()
    m = _model(c)
    try:
        m.set_tensor_cores(tc)
        out = _forward(m, _utt(meta), meta["seed"])
    finally:
        m.set_tensor_cores(True)
    e = {k: _maxabs(out[k], g[f"{c}/{k}"]) for k in ("mel_out", "pitch_pred", "decoder_inp", "style") if f"{c}/{k}" in g.files}
    e["spk"] = _maxabs(out["spk_proj"][0], g[f"{c}/spk_embed"])
    if m.hp["emo"]:
        e["emo"] = _maxabs(out["emo_proj"][0], g[f"{c}/emo_embed"])
    e_f0 = _maxabs(out["f0_denorm"], g[f"{c}/f0_denorm"])
    codes_ok = not m.hp["style"] or np.array_equal(out["rq_codes"].cpu().numpy(), g[f"{c}/rq_codes"])
    print(f"{c} ({'tc' if tc else 'ffma'}): " + ", ".join(f"{k} {v:.3e}" for k, v in e.items()) +
          f", f0_denorm {e_f0:.3e} Hz, rq codes exact {codes_ok}")
    assert codes_ok
    assert e["mel_out"] < 1e-3 and all(v < 1e-4 for k, v in e.items() if k != "mel_out")
    assert e_f0 < 5e-2
    if m.spk_id:  # the table row itself, copied
        assert _maxabs(out["spk_proj"][0], m_table(c)[meta["spk_id"]]) == 0.0


def m_table(c):
    return fft_spkid_sd(_cfg(c))["spk_embed_proj.weight"]


def test_duration_path_matches_reference_golden():
    g, meta = _fixture()
    c = meta["dur_config"]
    m = _model(c)
    out = _forward(m, _utt(meta), meta["seed"] + 1, use_mel2ph=False)
    e_mel = _maxabs(out["mel_out"], g[f"{c}/dur_mel_out"])
    e_f0 = _maxabs(out["f0_denorm"], g[f"{c}/dur_f0_denorm"])
    m2p_ok = np.array_equal(out["mel2ph"].cpu().numpy(), g[f"{c}/dur_mel2ph"])
    print(f"{c}, predicted durations: mel2ph exact {m2p_ok}, mel_out {e_mel:.3e}, f0_denorm {e_f0:.3e} Hz")
    assert m2p_ok and e_mel < 1e-3 and e_f0 < 5e-2


def _bench_utts(n, first=0, seed=1234):
    secs = synth.batch_seconds(64, seed=seed)[first:first + n]
    us = [synth.make_utterance(float(s), utt_idx=first + i, ref_frames=1125) for i, s in enumerate(secs)]
    for i, u in enumerate(us):
        u["spk_id"] = (7 * (first + i)) % 151
    return us


class _Noise64:
    """NoiseSource draws in float64, for the float64 oracle."""

    def __init__(self, seed):
        self.ns = O.NoiseSource(seed)

    def randn(self, shape):
        return self.ns.randn(shape).double()

    def rand(self, shape):
        return self.ns.rand(shape).double()


@pytest.mark.parametrize("c", ["fft_conv", "fft_gmdiff"])
def test_ragged_batch_at_bench_lengths_matches_oracle(c):
    """16 utterances of the batch64 workload (about 26 k frames: the tensor-core FFT decoder / attention paths), T = 4.
    fft + conv draws nothing; fft + gmdiff gets injected F0 noise.  The three shortest utterances are checked against the
    test oracle: the whole forward in float64 for fft + conv, and in fp32 for fft + gmdiff (the shared oracle's F0 sampler
    is fp32-only).  On every utterance, the FFT decoder + mel_out is checked in float64 on the kernel's own decoder_inp,
    which isolates the decoder from pitch-bin decisions."""
    T = 4
    m = _model(c, T)
    hp = m.hp
    utts = _bench_utts(16)
    lens = [len(u["mel2ph"]) for u in utts]
    pb = m.pack_batch(utts).to(DEV)
    noise = None
    if hp["f0_gen"] == "gmdiff":
        noise = _f0_noise([_noise(hp, 300 + i, lens[i]) for i in range(len(utts))])
    out = m.forward(pb, noise=noise, want=("mel_out", "decoder_inp", "pitch_pred", "f0_denorm"))
    torch.cuda.synchronize()
    fo = pb.frame_offsets
    sd = fft_spkid_sd(_cfg(c, T))
    sd64 = {k: v.double() for k, v in sd.items()}
    worst = {"decoder_inp": 0.0, "pitch_pred": 0.0, "mel_out(own decoder_inp)": 0.0}
    f64 = hp["f0_gen"] == "conv"
    flips = 0
    for i in np.argsort(lens)[:3]:
        u = utts[i]
        d = (lambda x: x.double()) if f64 else (lambda x: x)
        with torch.no_grad():
            r = O.stylesinger_forward(sd64 if f64 else sd, hp, u["txt_tokens"][None], u["note"][None],
                                      d(u["note_dur"][None]), u["note_type"][None], d(u["spk_embed"][None]),
                                      d(u["emo_embed"][None]), d(u["ref_mels"][None]), d(u["ref_f0"]),
                                      _Noise64(300 + i) if f64 else O.NoiseSource(300 + i), mel2ph=u["mel2ph"][None])
        # a coarse pitch bin decided the other way (f0 within rounding of a bin edge) changes that frame's pitch_embed row:
        # decoder_inp is compared on the frames whose bins agree, and at most 2 may disagree
        bins = O.f0_to_coarse(out["f0_denorm"][fo[i]:fo[i + 1]].double().cpu()).reshape(-1)
        same = (bins == r["pitch"][0].reshape(-1).to(bins)).to(DEV)
        flips += int((~same).sum())
        worst["decoder_inp"] = max(worst["decoder_inp"], _maxabs(out["decoder_inp"][fo[i]:fo[i + 1]][same], r["decoder_inp"][0][same.cpu()]))
        worst["pitch_pred"] = max(worst["pitch_pred"], _maxabs(out["pitch_pred"][fo[i]:fo[i + 1]][:, 0], r["pitch_pred"][0][:, 0]))
    for i in range(len(utts)):
        dec = out["decoder_inp"][fo[i]:fo[i + 1]].double().cpu()[None]
        tgt = (torch.as_tensor(utts[i]["mel2ph"]) > 0).double()[None, :, None]
        with torch.no_grad():
            mel = torch.nn.functional.linear(O.fastspeech_decoder(dec, sd64, hp), sd64["mel_out.weight"],
                                             sd64["mel_out.bias"]) * tgt
        worst["mel_out(own decoder_inp)"] = max(worst["mel_out(own decoder_inp)"], _maxabs(out["mel_out"][fo[i]:fo[i + 1]], mel[0]))
    print(f"{c}: {len(utts)} utterances, {int(fo[-1])} frames; " + ", ".join(f"{k} {v:.3e}" for k, v in worst.items()) +
          f", coarse-bin flips {flips}")
    assert flips <= 2 and worst["decoder_inp"] < 1e-3 and worst["pitch_pred"] < 1e-3 and worst["mel_out(own decoder_inp)"] < 1e-3


def _drop(sd, prefixes):
    return {k: v for k, v in sd.items() if not k.startswith(prefixes)}


@pytest.mark.parametrize("f0_gen", ["gmdiff", "conv"])
def test_fft_model_is_the_diffsinger_models_coarse_mel(f0_gen):
    """An FFT model and a DiffSinger model built from the same weights: the FFT model's mel_out is bitwise the DiffSinger
    model's coarse_mel, and decoder_inp, f0_denorm, pitch_pred and mel2ph are bitwise equal, for the same inputs and F0
    noise (short batches on FFMA, a long one on the tensor-core decoder path)."""
    from stylesinger_b200.engine import AcousticModel
    T = 4
    hp_d = fft_spkid_hp({"T": T, "overrides": {"f0_gen": f0_gen}})
    hp_f = fft_spkid_hp({"T": T, "overrides": {"f0_gen": f0_gen, "decoder": "fft"}})
    sd_d = fft_spkid_sd({"T": T, "overrides": {"f0_gen": f0_gen}})
    a = AcousticModel(sd_d, hp_d, DEV)
    b = AcousticModel(_drop(sd_d, ("postdiff.", "ln_proj.")), hp_f, DEV)
    for utts in ([synth.make_utterance(0.3 + 0.2 * i, utt_idx=i, ref_frames=40 + 9 * i) for i in range(3)], _bench_utts(8)):
        lens = [len(u["mel2ph"]) for u in utts]
        noise = None
        if f0_gen == "gmdiff":
            noise = _f0_noise([_noise(hp_f, 50 + i, n) for i, n in enumerate(lens)])
        keys = ("decoder_inp", "f0_denorm", "pitch_pred", "mel2ph")
        oa = a.forward(a.pack_batch(utts).to(DEV), noise=noise, skip_mel_diffusion=True, want=keys + ("coarse_mel",))
        ob = b.forward(b.pack_batch(utts).to(DEV), noise=noise, want=keys + ("mel_out", "coarse_mel"))
        torch.cuda.synchronize()
        assert torch.equal(oa["coarse_mel"], ob["mel_out"]) and torch.equal(ob["coarse_mel"], ob["mel_out"])
        for k in keys:
            assert torch.equal(oa[k], ob[k]), k
        print(f"{f0_gen}: {sum(lens)} frames, FFT mel_out == DiffSinger coarse_mel bitwise")


@pytest.mark.parametrize("dec", ["diffsinger", "prodiff", "fft"])
def test_speaker_table_equals_the_linear_projection(dec):
    """A use_spk_id model whose table rows are the spk_proj outputs of a Linear model gives bitwise that model's outputs."""
    from stylesinger_b200.engine import AcousticModel
    T = 4
    ov = {"decoder": dec, **({"schedule_type": "vpsde"} if dec == "prodiff" else {})}
    hp = fft_spkid_hp({"T": T, "overrides": ov})
    hp_id = fft_spkid_hp({"T": T, "overrides": dict(ov, use_spk_id=True)})
    sd = fft_spkid_sd({"T": T, "overrides": ov})
    lin = AcousticModel(sd, hp, DEV)
    utts = [synth.make_utterance(0.3 + 0.1 * i, utt_idx=20 + i, ref_frames=40) for i in range(4)]
    ids = [5, 150, 0, 77]
    spk = lin.forward(lin.pack_batch(utts).to(DEV), seed=3, want=("spk_proj",), skip_mel_diffusion=True)["spk_proj"].cpu()
    table = torch.zeros(151, 256)
    for i, r in zip(ids, spk):
        table[i] = r
    sd_id = _drop(sd, ("spk_embed_proj.",))
    sd_id["spk_embed_proj.weight"] = table
    mid = AcousticModel(sd_id, hp_id, DEV)
    for u, i in zip(utts, ids):
        u["spk_id"] = i
    want = ("mel_out", "f0_denorm", "decoder_inp", "pitch_pred", "spk_proj", "style", "rq_codes")
    oa = lin.forward(lin.pack_batch(utts).to(DEV), seed=11, want=want)
    ob = mid.forward(mid.pack_batch(utts).to(DEV), seed=11, want=want)
    torch.cuda.synchronize()
    for k in want:
        assert torch.equal(oa[k], ob[k]), k
    pa, pb_ = lin.pack_batch(utts).to(DEV), mid.pack_batch(utts).to(DEV)
    assert torch.equal(lin.predict_durations(pa)[0], mid.predict_durations(pb_)[0])
    print(f"{dec}: use_spk_id model == Linear model bitwise on {len(want)} outputs and the durations")


def _launches():
    from stylesinger_b200._lib import lib
    return int(lib.ssb_launch_count())


def test_documented_errors_launch_nothing():
    from stylesinger_b200._lib import AcousticOutputs, SsbError, lib
    m = _model("spkid_fft")
    u = dict(synth.make_utterance(0.2, utt_idx=1, ref_frames=20, frames=30, phones=5), spk_id=3)
    pb = m.pack_batch([u]).to(DEV)
    mel = torch.empty(30, 80, device=DEV)
    torch.cuda.synchronize()

    def refused(fn, cause):
        n0 = _launches()
        with pytest.raises(SsbError, match=cause):
            fn()
        assert _launches() == n0, cause

    for ids, cause in (([151], r"spk_ids\[0\] = 151 is outside \[0, 151\)"), ([-1], r"spk_ids\[0\] = -1 is outside"),
                       (None, "needs spk_ids")):
        pb.spk_ids = None if ids is None else np.array(ids, np.int32)
        refused(lambda: m.forward(pb, seed=0, want=("mel_out",)), cause)
        refused(lambda: m.forward(pb, seed=0, want=("mel_out",), seeds=[1]), cause)
        refused(lambda: m.predict_durations(pb), cause)
    pb.spk_ids = np.array([3], np.int32)
    # the library's own checks of an FFT model, below the host-side ones of AcousticModel.forward
    from stylesinger_b200.engine import _ptr
    a = m._inputs(pb)
    o = AcousticOutputs()
    o.mel_out = mel.data_ptr()
    ws = m._ws.get(int(lib.ssb_acoustic_workspace_bytes(m._h, C.byref(a))))
    stream = m._stream()
    o.diff_cond = torch.empty(30, 256, device=DEV).data_ptr()
    n0 = _launches()
    assert lib.ssb_acoustic_forward(m._h, C.byref(a), C.byref(o), _ptr(ws), ws.numel(), stream) != 0
    assert "no diff_cond" in lib.ssb_last_error().decode() and _launches() == n0
    o.diff_cond = None
    a.mel_noise = torch.zeros(5, 30, 80, device=DEV).data_ptr()
    assert lib.ssb_acoustic_forward(m._h, C.byref(a), C.byref(o), _ptr(ws), ws.numel(), stream) != 0
    assert "draws no mel noise" in lib.ssb_last_error().decode() and _launches() == n0
    with pytest.raises(SsbError, match="no diff_cond"):
        m.forward(pb, seed=0, want=("mel_out", "diff_cond"))
    fo = np.array([0, 30], np.int32)
    cond, x = torch.zeros(30, 256, device=DEV), torch.zeros(30, 80, device=DEV)
    refused(lambda: m.set_timesteps(4), "no mel diffusion schedule")
    for K in (0, 4):
        refused(lambda: m.set_mel_k_step(K), "no mel sampler and no K_step")
    refused(lambda: m.mel_diffusion(cond, x, fo), "ssb_mel_diffusion_sample: a model with the FFT mel decoder")
    refused(lambda: m.mel_diffusion_plms(cond, x, fo, 2), "ssb_mel_diffusion_sample_plms: a model with the FFT mel decoder")
    refused(lambda: m.mel_prodiff(cond, fo), "ssb_mel_prodiff_sample: a model with the FFT mel decoder")
    refused(lambda: m.denoiser_eval(0, x, None, 0, cond, fo), "has no mel DiffNet")
    m.set_mel_precision("fp16")  # accepted, changes nothing: there is no mel DiffNet
    try:
        out = m.forward(pb, seed=0, want=("mel_out",))
    finally:
        m.set_mel_precision("split")
    ref = m.forward(pb, seed=0, want=("mel_out",))
    torch.cuda.synchronize()
    assert torch.equal(out["mel_out"], ref["mel_out"])
    # a table whose rows do not match num_spk
    from stylesinger_b200.engine import AcousticModel
    with pytest.raises(ValueError, match="num_spk"):
        AcousticModel(fft_spkid_sd(_cfg("spkid_fft")), dict(fft_spkid_hp(_cfg("spkid_fft")), num_spk=20), DEV)


@pytest.mark.parametrize("c", ["fft_gmdiff", "spkid_diffsinger", "spkid_fft"])
def test_workspace_dry_run_matches_the_real_run(c):
    from stylesinger_b200._lib import lib
    m = _model(c)
    utts = _bench_utts(4)
    pb = m.pack_batch(utts).to(DEV)
    n = lib.ssb_acoustic_workspace_bytes(m._h, C.byref(m._inputs(pb)))
    assert n > 0
    m._ws.buf = torch.empty(n, dtype=torch.uint8, device=DEV)  # exactly the dry run's size
    out = m.forward(pb, seed=1, want=("mel_out",))
    nd = lib.ssb_durations_workspace_bytes(m._h, C.byref(m._inputs(pb)))
    m._ws.buf = torch.empty(nd, dtype=torch.uint8, device=DEV)
    m.predict_durations(pb)
    torch.cuda.synchronize()
    assert torch.isfinite(out["mel_out"]).all()
    if m.mel_decoder == "fft":  # no cond / cat / sampler buffers: less than the DiffSinger model of the same switches
        d = _model("spkid_diffsinger")
        nd = lib.ssb_acoustic_workspace_bytes(d._h, C.byref(d._inputs(d.pack_batch(utts).to(DEV))))
        print(f"{c}: workspace {n / 2**20:.1f} MiB, DiffSinger {nd / 2**20:.1f} MiB")
        assert n < nd


def test_keyed_utterances_equal_their_solo_calls_with_ffma():
    m = _model("fft_gmdiff")
    utts = _bench_utts(6, first=10)
    seeds = [1000 + 7 * i for i in range(len(utts))]
    want = ("mel_out", "f0_denorm", "decoder_inp")
    try:
        m.set_tensor_cores(False)
        m.set_persistent(False)
        pb = m.pack_batch(utts).to(DEV)
        batch = m.forward(pb, seeds=seeds, want=want)
        fo = pb.frame_offsets
        for b, u in enumerate(utts):
            solo = m.forward(m.pack_batch([u]).to(DEV), seed=seeds[b], want=want)
            for k in want:
                assert torch.equal(batch[k][fo[b]:fo[b + 1]], solo[k]), (b, k)
    finally:
        m.set_tensor_cores(True)
        m.set_persistent(True)


def test_padding_frames_are_zero_and_dropped_before_the_vocoder():
    """On an FFT model, frames with mel2ph = 0 (an interior gap and a padded tail) come out exactly 0 (tgt_nonpadding), and
    StyleSingerInfer drops them before the vocoder, as the reference drops all-zero frames (inference/StyleSinger.py:56-62)."""
    from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG
    from stylesinger_b200.infer import StyleSingerInfer
    hp = fft_spkid_hp({"T": 4, "overrides": {"decoder": "fft", "f0_gen": "conv"}})
    inf = StyleSingerInfer(hp, DEV, fft_spkid_sd({"T": 4, "overrides": {"decoder": "fft", "f0_gen": "conv"}}),
                           synth.vocoder_state_dict(DEFAULT_VOCODER_CONFIG, seed=0), DEFAULT_VOCODER_CONFIG)
    utts = [synth.make_utterance(0.5 + 0.2 * i, utt_idx=30 + i, ref_frames=48) for i in range(2)]
    for u in utts:
        m2p = u["mel2ph"].clone()
        m2p[40:52] = 0
        u["mel2ph"] = torch.cat([m2p, torch.zeros(10, dtype=m2p.dtype)])
    pb = inf.model.pack_batch(utts).to(DEV)
    mel, f0, wav, fo_v = inf.run_device(pb, seed=0)
    torch.cuda.synchronize()
    keep = torch.cat([u["mel2ph"] > 0 for u in utts]).to(DEV)
    assert torch.all(mel[~keep] == 0) and bool((mel[keep].abs().sum(-1) > 0).all())
    assert fo_v.tolist() == np.concatenate([[0], np.cumsum([int((u["mel2ph"] > 0).sum()) for u in utts])]).tolist()
    assert wav.numel() == int(fo_v[-1]) * inf.vocoder.hop and torch.isfinite(wav).all()
