"""Model switches (hparams emo / style / umln / use_txt_cond) on the CUDA path: every configuration of
tests/golden/ref_switches.npz against the unmodified reference on FFMA and on tensor cores, ragged batches at bench
lengths against the test oracle, ssb_model_create_ex3 with every switch on against ssb_model_create_ex2, the work a
style-off forward skips, keyed seeds, the workspace dry run and the documented errors."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from tests.common import batch_noise, engine_noise_from_stream, golden, switch_hp, switch_sd, utt_from_meta

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_C = {}
CONFIGS = ("no_emo", "no_style", "no_umln", "no_txt_cond", "all_off", "prodiff_no_emo_style", "conv_no_style")


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    """The models this module caches hold their packed weights and their largest workspace (several GB after the
    bench-length batches): free them when the module ends, so that the modules after it in the same process get the
    device memory back."""
    yield
    _C.clear()
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    print(f"after test_gpu_switches: {torch.cuda.memory_allocated() / 2**30:.2f} GiB allocated by torch, "
          f"{torch.cuda.mem_get_info()[0] / 2**30:.1f} GiB free on the device")


def _maxabs(a, b):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def _fixture():
    if "g" not in _C:
        _C["g"], _C["meta"] = golden("ref_switches")
    return _C["g"], _C["meta"]


def _cfg(c, T=None):
    _, meta = _fixture()
    return {"T": T or meta["T"], "overrides": meta["configs"][c]["overrides"]}


def _model(c, T=None):
    from stylesinger_b200.engine import AcousticModel
    key = (c, T)
    if key not in _C:
        _C[key] = AcousticModel(switch_sd(_cfg(c, T)), switch_hp(_cfg(c, T)), DEV)
    m = _C[key]
    m.set_tensor_cores(True)
    m.set_persistent(True)
    m.set_persistent_groups(False)
    return m


def _noise(hp, seed, Fr):
    """The forward's draws from NoiseSource(seed) in the C ABI's layout: the two F0 samplers' (gmdiff) then the mel
    sampler's T + 1."""
    T = hp["timesteps"]
    if hp["f0_gen"] == "conv":
        ns = O.NoiseSource(seed)
        return {"mel": torch.stack([ns.randn((1, 1, 80, Fr))[0, 0].t() for _ in range(T + 1)]).contiguous().to(DEV)}
    return engine_noise_from_stream(seed, T, T, Fr, DEV)[0]


def _want(hp):
    w = ["mel_out", "f0_denorm", "pitch_pred", "decoder_inp", "mel2ph", "spk_proj"]
    w += ["emo_proj"] if hp["emo"] else []
    w += ["style", "rq_codes"] if hp["style"] else []
    return tuple(w)


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
        out = _forward(m, utt_from_meta(meta), meta["seed"])
    finally:
        m.set_tensor_cores(True)
    e = {k: _maxabs(out[k], g[f"{c}/{k}"]) for k in ("mel_out", "pitch_pred", "decoder_inp", "style")
         if f"{c}/{k}" in g.files}
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


def test_duration_path_matches_reference_golden():
    g, meta = _fixture()
    c = meta["dur_config"]
    m = _model(c)
    out = _forward(m, utt_from_meta(meta), meta["seed"] + 1, use_mel2ph=False)
    e_mel = _maxabs(out["mel_out"], g[f"{c}/dur_mel_out"])
    e_f0 = _maxabs(out["f0_denorm"], g[f"{c}/dur_f0_denorm"])
    m2p_ok = np.array_equal(out["mel2ph"].cpu().numpy(), g[f"{c}/dur_mel2ph"])
    print(f"{c}, predicted durations: mel2ph exact {m2p_ok}, mel_out {e_mel:.3e}, f0_denorm {e_f0:.3e} Hz")
    assert m2p_ok and e_mel < 1e-3 and e_f0 < 5e-2


def _bench_utts(n, first=0, seed=1234):
    secs = synth.batch_seconds(64, seed=seed)[first:first + n]
    return [synth.make_utterance(float(s), utt_idx=first + i, ref_frames=1125) for i, s in enumerate(secs)]


@pytest.mark.parametrize("c", ["no_style", "all_off"])
def test_ragged_batch_at_bench_lengths_matches_oracle(c):
    """16 utterances of the batch64 workload (about 26 k frames: the tensor-core FFT FFN / attention paths), T = 4 with
    injected noise; the three shortest utterances are checked against the test oracle, and the batch against its
    own persistent-group run (Philox) for finiteness."""
    T = 4
    m = _model(c, T)
    utts = _bench_utts(16)
    hp = m.hp
    lens = [len(u["mel2ph"]) for u in utts]
    per = [_noise(hp, 300 + i, lens[i]) for i in range(len(utts))]
    pb = m.pack_batch(utts).to(DEV)
    out = m.forward(pb, noise=batch_noise(per) if hp["f0_gen"] == "gmdiff" else
                    {"mel": torch.cat([n["mel"] for n in per], 1).contiguous()}, want=("mel_out", "decoder_inp", "f0_denorm"))
    fo = pb.frame_offsets
    worst = {"mel_out": 0.0, "decoder_inp": 0.0}
    for i in np.argsort(lens)[:3]:
        u = utts[i]
        ns = O.NoiseSource(300 + i)
        with torch.no_grad():
            r = O.stylesinger_forward(switch_sd(_cfg(c, T)), hp, u["txt_tokens"][None], u["note"][None],
                                      u["note_dur"][None], u["note_type"][None], u["spk_embed"][None],
                                      u["emo_embed"][None], u["ref_mels"][None], u["ref_f0"], ns,
                                      mel2ph=u["mel2ph"][None])
        for k in worst:
            worst[k] = max(worst[k], _maxabs(out[k][fo[i]:fo[i + 1]], r[k][0]))
    print(f"{c}: {len(utts)} utterances, {int(fo[-1])} frames; worst of 3 vs oracle: "
          + ", ".join(f"{k} {v:.3e}" for k, v in worst.items()))
    assert worst["decoder_inp"] < 1e-3 and worst["mel_out"] < 5e-3
    m.set_persistent_groups(True)
    try:
        o2 = m.forward(pb, seed=5, want=("mel_out",))
        torch.cuda.synchronize()
    finally:
        m.set_persistent_groups(False)
    assert torch.isfinite(o2["mel_out"]).all()


def test_ex3_with_every_switch_on_is_ex2_bitwise():
    from stylesinger_b200._lib import check, lib
    from stylesinger_b200.engine import AcousticModel
    hp = switch_hp({"T": 4, "overrides": {}})
    sd = synth.acoustic_state_dict(hp, seed=0)
    a = AcousticModel(sd, hp, DEV)  # ex3 (all on)
    b = AcousticModel(sd, hp, DEV)
    h = C.c_void_p()
    from stylesinger_b200.engine import HParams, _descs, sinusoid_table  # noqa: F401
    # swap b's model for one created through ssb_model_create_ex2
    sd2 = dict(sd, __pos_table=sinusoid_table(4096, 256))
    sd2["encoder.embed_tokens.weight"] = sd["encoder_embed_tokens.weight"]
    arr, keep = _descs(sd2)
    hh = HParams(256, hp["enc_layers"], hp["dec_layers"], hp["enc_ffn_kernel_size"], hp["dec_ffn_kernel_size"],
                 hp["dur_predictor_layers"], hp["dur_predictor_kernel"], int(sd["encoder_embed_tokens.weight"].shape[0]),
                 hp["nRQ"], hp["rq_depth"], hp["residual_channels"], hp["residual_layers"], hp["dilation_cycle_length"],
                 hp["f0_residual_channels"], hp["f0_residual_layers"], hp["f0_dilation_cycle_length"], 80)
    check(lib.ssb_model_create_ex2(C.byref(h), arr, len(sd2), C.byref(hh), 0, 0), "ssb_model_create_ex2")
    lib.ssb_model_free(b._h)
    b._h = h
    b.T = b.f0_T = None
    b.set_timesteps(4, 4)
    utts = [synth.make_utterance(0.3 + 0.2 * i, utt_idx=i, ref_frames=40 + 9 * i) for i in range(3)]
    want = ("mel_out", "f0_denorm", "encoder_out", "style", "rq_codes", "pitch_pred", "decoder_inp", "coarse_mel",
            "diff_cond", "mel2ph", "spk_proj", "emo_proj")
    for tc in (False, True):
        outs = []
        for m in (a, b):
            m.set_tensor_cores(tc)
            outs.append(m.forward(m.pack_batch(utts).to(DEV), seed=77, want=want))
            m.set_tensor_cores(True)
        torch.cuda.synchronize()
        for k in want:
            assert torch.equal(outs[0][k], outs[1][k]), (tc, k)
        print(f"tensor cores {tc}: ex3 (all on) == ex2 bitwise on {len(want)} outputs")


def test_style_off_runs_no_aligner_and_no_rvq():
    from stylesinger_b200._lib import lib
    m = _model("all_off")
    utts = _bench_utts(4)
    pb = m.pack_batch(utts).to(DEV)
    assert "ref_mels" not in pb.t and pb.ref_offsets is None
    a0, a1, n0 = lib.ssb_attention_launch_count(0), lib.ssb_attention_launch_count(1), lib.ssb_launch_count()
    out = m.forward(pb, seed=3, want=("mel_out",))
    torch.cuda.synchronize()
    n_all_off = lib.ssb_launch_count() - n0
    att_off = (lib.ssb_attention_launch_count(0) - a0) + (lib.ssb_attention_launch_count(1) - a1)
    # the FFT blocks still attend (self-attention): count what the default model launches on the same batch
    d = _C.get("default") or _model_default()
    pbd = d.pack_batch(utts).to(DEV)
    b0, b1, m0 = lib.ssb_attention_launch_count(0), lib.ssb_attention_launch_count(1), lib.ssb_launch_count()
    d.forward(pbd, seed=3, want=("mel_out",))
    torch.cuda.synchronize()
    att_on = (lib.ssb_attention_launch_count(0) - b0) + (lib.ssb_attention_launch_count(1) - b1)
    n_on = lib.ssb_launch_count() - m0
    print(f"attention launches: all off {att_off}, default {att_on} (2 aligner layers); kernel launches {n_all_off} vs {n_on}")
    assert att_on - att_off == 2  # the ProsodyAligner's two cross-attention layers
    assert torch.isfinite(out["mel_out"]).all()
    # the style-off model refuses the style entry points and outputs
    with pytest.raises(Exception, match="style"):
        m.get_style(torch.zeros(10, 256, device=DEV), np.array([0, 10], np.int32), torch.zeros(10, 80, device=DEV),
                    torch.zeros(10, device=DEV), np.array([0, 10], np.int32))
    with pytest.raises(Exception, match="style"):
        m.rvq(torch.zeros(10, 256, device=DEV), np.array([0, 10], np.int32))
    for k in ("style", "rq_codes", "emo_proj"):
        with pytest.raises(Exception, match="emo|style"):
            m.forward(pb, seed=3, want=("mel_out", k))


def _model_default():
    from stylesinger_b200.engine import AcousticModel
    hp = switch_hp({"T": 4, "overrides": {}})
    _C["default"] = AcousticModel(synth.acoustic_state_dict(hp, seed=0), hp, DEV)
    return _C["default"]


@pytest.mark.parametrize("c", ["no_style", "all_off", "prodiff_no_emo_style", "conv_no_style"])
def test_keyed_utterances_equal_their_solo_calls_with_ffma(c):
    m = _model(c)
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
                assert torch.equal(batch[k][fo[b]:fo[b + 1]], solo[k]), (c, b, k)
    finally:
        m.set_tensor_cores(True)
        m.set_persistent(True)
    print(f"{c}: {len(utts)} keyed utterances bitwise equal to their solo calls (FFMA)")


@pytest.mark.parametrize("c", ["no_style", "all_off", "prodiff_no_emo_style"])
def test_workspace_dry_run_matches_the_real_run(c):
    """The workspace the dry run sizes is enough, and the style-off dry run takes less than the default model's."""
    from stylesinger_b200._lib import lib
    m = _model(c)
    utts = _bench_utts(4)
    pb = m.pack_batch(utts).to(DEV)
    a = m._inputs(pb)
    n = lib.ssb_acoustic_workspace_bytes(m._h, C.byref(a))
    assert n > 0
    m._ws.buf = torch.empty(n, dtype=torch.uint8, device=DEV)  # exactly the dry run's size
    out = m.forward(pb, seed=1, want=("mel_out",))
    torch.cuda.synchronize()
    assert torch.isfinite(out["mel_out"]).all()
    d = _C.get("default") or _model_default()
    nd = lib.ssb_acoustic_workspace_bytes(d._h, C.byref(d._inputs(d.pack_batch(utts).to(DEV))))
    print(f"{c}: workspace {n / 2**20:.1f} MiB (default model {nd / 2**20:.1f} MiB)")
    if not m.hp["style"]:
        assert n < nd


def test_documented_errors():
    from stylesinger_b200._lib import SsbError
    m = _model("all_off")
    u = synth.make_utterance(0.2, utt_idx=1, ref_frames=20, frames=30, phones=5)
    pb = m.pack_batch([u]).to(DEV)
    for k, cause in (("emo_proj", "without emo"), ("style", "without style"), ("rq_codes", "without style")):
        with pytest.raises(SsbError, match=cause):
            m.forward(pb, seed=0, want=("mel_out", k))
    with pytest.raises(SsbError, match="without style"):
        m.get_style(torch.zeros(30, 256, device=DEV), np.array([0, 30], np.int32), torch.zeros(20, 80, device=DEV),
                    torch.zeros(20, device=DEV), np.array([0, 20], np.int32))
    with pytest.raises(SsbError, match="without style"):
        m.rvq(torch.zeros(20, 256, device=DEV), np.array([0, 20], np.int32))
    # a checkpoint whose ln_proj does not match the switches
    from stylesinger_b200.engine import AcousticModel
    hp = switch_hp(_cfg("no_emo"))
    with pytest.raises(SsbError, match=r"ln_proj.weight must be \[256, 848\]"):
        AcousticModel(synth.acoustic_state_dict(switch_hp({"T": 4, "overrides": {}}), seed=0), hp, DEV)
    # the emo-off model works without emo_embed in the batch, the style-off one without reference mels
    out = m.forward(pb, seed=0, want=("mel_out",))
    assert torch.isfinite(out["mel_out"]).all()
