"""The FastSpeech 2 mel decoder (decoder: fft) and speaker ids (use_spk_id), CPU side: the test oracle and the synthetic
checkpoints against the unmodified reference (tests/golden/ref_fft_spkid.npz), the hparams rules, the C ABI's argument
checks (no GPU needed) and the host-side batch packing of speaker ids."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from stylesinger_b200.engine import pack_batch
from stylesinger_b200.hparams import resolve
from tests.common import fft_spkid_hp, fft_spkid_sd, golden, switch_sd, utt_from_meta

TOL = 2e-5  # fp32 CPU, same op order up to BLAS blocking (as tests/test_switches_cpu.py)
CONFIGS = ("fft_gmdiff", "fft_conv", "spkid_diffsinger", "spkid_fft", "fft_no_emo_style")


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def _cfg(meta, c):
    return {"T": meta["T"], "overrides": meta["configs"][c]["overrides"]}


def _spk(meta, hp, u):
    """The speaker input of the fixture's forwards: the id meta['spk_id'] with use_spk_id, else the speaker vector."""
    return torch.tensor([meta["spk_id"]]) if hp["use_spk_id"] else u["spk_embed"][None]


def _forward(meta, c, seed, use_mel2ph=True):
    cfg = _cfg(meta, c)
    hp = fft_spkid_hp(cfg)
    u = utt_from_meta(meta)
    ns = O.NoiseSource(seed)
    with torch.no_grad():
        r = O.stylesinger_forward(fft_spkid_sd(cfg), hp, u["txt_tokens"][None], u["note"][None], u["note_dur"][None],
                                  u["note_type"][None], _spk(meta, hp, u), u["emo_embed"][None], u["ref_mels"][None],
                                  u["ref_f0"], ns, mel2ph=u["mel2ph"][None] if use_mel2ph else None)
    return r, ns


def test_fixture_covers_every_configuration():
    g, meta = golden("ref_fft_spkid")
    assert tuple(meta["configs"]) == CONFIGS
    seen = set()
    for c in CONFIGS:
        hp = fft_spkid_hp(_cfg(meta, c))
        seen.add((hp["decoder"], hp["f0_gen"], hp["use_spk_id"], hp["emo"] and hp["style"]))
        assert (f"{c}/style" in g.files) == hp["style"] and (f"{c}/emo_embed" in g.files) == hp["emo"]
        assert (f"{c}/coarse_mel" in g.files) == (hp["decoder"] == "diffsinger")
    # fft x {gmdiff, conv}; use_spk_id on a DiffSinger and on an FFT model; an FFT model with emo / style off
    for want in (("fft", "gmdiff", False, True), ("fft", "conv", False, True), ("diffsinger", "gmdiff", True, True),
                 ("fft", "gmdiff", True, True), ("fft", "gmdiff", False, False)):
        assert want in seen, want
    assert fft_spkid_hp(_cfg(meta, meta["dur_config"]))["use_spk_id"]


@pytest.mark.parametrize("c", CONFIGS)
def test_oracle_forward_matches_reference(c):
    g, meta = golden("ref_fft_spkid")
    r, ns = _forward(meta, c, meta["seed"])
    assert [[k, list(sh)] for k, sh in ns.log] == meta["configs"][c]["noise_log"]  # same draws in the same order
    errs = {}
    for k in ("mel_out", "pitch_pred", "decoder_inp", "spk_embed", "emo_embed", "style", "coarse_mel"):
        if f"{c}/{k}" in g.files:
            errs[k] = _maxabs(r[k][0].numpy(), g[f"{c}/{k}"])
    errs["f0_denorm(Hz)"] = _maxabs(r["f0_denorm"][0].numpy(), g[f"{c}/f0_denorm"])
    print(c, errs)
    assert all(v < TOL for k, v in errs.items() if k != "f0_denorm(Hz)"), errs
    assert errs["f0_denorm(Hz)"] < 1e-3
    if f"{c}/rq_codes" in g.files:
        assert np.array_equal(r["rq_codes"][0].numpy(), g[f"{c}/rq_codes"])  # RVQ indices: bit-exact
    if fft_spkid_hp(_cfg(meta, c))["decoder"] == "fft":
        assert "coarse_mel" not in r and "diff_cond" not in r


def test_oracle_duration_path_matches_reference():
    g, meta = golden("ref_fft_spkid")
    c = meta["dur_config"]
    r, ns = _forward(meta, c, meta["seed"] + 1, use_mel2ph=False)
    assert [[k, list(sh)] for k, sh in ns.log] == meta["configs"][c]["dur_noise_log"]
    assert np.array_equal(r["mel2ph"][0].numpy(), g[f"{c}/dur_mel2ph"])  # integer path: bit-exact
    e = {"logdur": _maxabs(r["dur"][0].numpy(), g[f"{c}/dur_logdur"]),
         "mel_out": _maxabs(r["mel_out"][0].numpy(), g[f"{c}/dur_mel_out"])}
    print(c, e)
    assert max(e.values()) < TOL
    assert _maxabs(r["f0_denorm"][0].numpy(), g[f"{c}/dur_f0_denorm"]) < 1e-3


@pytest.mark.parametrize("c", CONFIGS)
def test_synth_keys_and_shapes_are_the_references(c):
    _, meta = golden("ref_fft_spkid")
    hp = fft_spkid_hp(_cfg(meta, c))
    ref = [[k, list(s)] for k, s in meta["configs"][c]["state_dict"]]
    assert [[k, list(s)] for k, s in synth.acoustic_param_shapes(hp)] == ref
    sd = fft_spkid_sd(_cfg(meta, c))
    assert [[k, list(v.shape)] for k, v in sd.items()] == ref
    keys = set(sd)
    if hp["decoder"] == "fft":
        assert not any(k.startswith(("postdiff.", "ln_proj.", "diff_decoder.")) for k in keys)
    if hp["use_spk_id"]:
        assert sd["spk_embed_proj.weight"].shape == (hp["num_spk"] + 1, 256) and "spk_embed_proj.bias" not in keys


def test_default_synthetic_checkpoint_is_byte_identical_to_the_switch_configurations():
    """The options off leave the synthetic checkpoints as they were: the default one and an emo-off one equal, tensor for
    tensor, those built with the options spelled out."""
    for ov in ({}, {"emo": False}):
        a = switch_sd({"T": 4, "overrides": ov})
        b = synth.acoustic_state_dict(resolve(timesteps=4, K_step=4, f0_timesteps=4, decoder="diffsinger",
                                              use_spk_id=False, use_spk_embed=True, **ov), seed=0)
        assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)


X = {"extended_models": True}  # the opt-in the two options need


def test_resolve_needs_the_opt_in_for_either_option():
    """decoder 'fft' and use_spk_id lie outside the egs/stylesinger.yaml model family: resolve refuses them, naming the
    option and the opt-in, unless hparams['extended_models'] is True; the opt-in changes nothing else."""
    for kw, name in (({"decoder": "fft"}, "decoder: fft"), ({"use_spk_id": True}, "use_spk_id: True"),
                     ({"decoder": "fft", "emo": False}, "decoder: fft"), ({"use_spk_id": True, "style": False}, "use_spk_id")):
        with pytest.raises(NotImplementedError, match="extended_models") as e:
            resolve(**kw)
        assert name in str(e.value)
        assert resolve(**kw, **X)["extended_models"] is True
    assert resolve()["extended_models"] is False
    base, opted = resolve(), resolve(**X)
    assert {k for k in base if base[k] != opted[k]} == {"extended_models"}
    for bad in (1, "yes", None):
        with pytest.raises(NotImplementedError, match="extended_models"):
            resolve(extended_models=bad)


def test_resolve_accepts_the_fft_decoder_and_ignores_the_diffusion_keys():
    """decoder 'fft' reads no timesteps, K_step, pndm_speedup or schedule_type: values the DiffSinger decoder refuses
    pass, as the ProDiff decoder's do."""
    assert resolve(decoder="fft", **X)["decoder"] == "fft"
    hp = resolve(decoder="fft", timesteps=8, K_step=1000, pndm_speedup=10, schedule_type="vpsde", f0_gen="conv",
                 emo=False, style=False, **X)
    assert hp["K_step"] == 1000 and hp["pndm_speedup"] == 10
    with pytest.raises(ValueError):
        resolve(timesteps=8, K_step=1000, **X)
    with pytest.raises(NotImplementedError):
        resolve(schedule_type="vpsde", **X)
    for bad in ("FFT", "wavenet", None):
        with pytest.raises(NotImplementedError, match="decoder"):
            resolve(decoder=bad, **X)


def test_resolve_speaker_inputs():
    """use_spk_id True takes either use_spk_embed (the Embedding wins, fs2.py:37-43); with both False the reference
    builds no spk_embed_proj and is refused; use_spk_id takes booleans only."""
    for emb in (True, False):
        for dec in ("diffsinger", "prodiff", "fft"):
            extra = {"schedule_type": "vpsde"} if dec == "prodiff" else {}
            hp = resolve(use_spk_id=True, use_spk_embed=emb, decoder=dec, **extra, **X)
            assert hp["use_spk_id"] is True and hp["num_spk"] == 150
    assert resolve(use_spk_id=True, f0_gen="conv", emo=False, style=False, **X)["use_spk_id"]
    with pytest.raises(NotImplementedError, match="both False"):
        resolve(use_spk_id=False, use_spk_embed=False, **X)
    for bad in (1, "yes"):
        with pytest.raises(NotImplementedError, match="use_spk_id"):
            resolve(use_spk_id=bad, **X)


def _create_ex4(mel_decoder=0, f0_gen=0, use_spk_id=0):
    from stylesinger_b200._lib import HParams, ModelSwitches, lib
    h = C.c_void_p()
    rc = lib.ssb_model_create_ex4(C.byref(h), None, 0, C.byref(HParams(hidden_size=256)), mel_decoder, f0_gen,
                                  C.byref(ModelSwitches(1, 1, 1, 1)), use_spk_id)
    return rc, h.value, lib.ssb_last_error().decode()


@pytest.mark.parametrize("flag", [2, -1, 7])
def test_model_create_ex4_rejects_a_bad_spk_id_flag_without_a_gpu(flag):
    rc, h, err = _create_ex4(use_spk_id=flag)
    print(flag, "rc", rc, "message:", err)
    assert rc != 0 and not h and f"use_spk_id must be 0 or 1, got {flag}" in err


@pytest.mark.parametrize("dec", [3, -1])
def test_model_create_ex4_rejects_an_unknown_decoder_without_a_gpu(dec):
    rc, h, err = _create_ex4(mel_decoder=dec)
    print(dec, "rc", rc, "message:", err)
    assert rc != 0 and not h and f"unknown mel_decoder {dec}" in err and "SSB_MEL_DECODER_FFT = 2" in err


def test_version_and_export():
    from stylesinger_b200._lib import EXPORTS, lib
    assert lib.ssb_version() >= 104 and "ssb_model_create_ex4" in EXPORTS


def _utts(n=3):
    us = [synth.make_utterance(0.2, utt_idx=i, ref_frames=16 + i, frames=30 + i, phones=5) for i in range(n)]
    for i, u in enumerate(us):
        u["spk_id"] = 10 * i + 3
    return us


def test_pack_batch_carries_host_speaker_ids():
    us = _utts()
    full = pack_batch(us)
    assert "spk_embed" in full.t and full.spk_ids is None
    pb = pack_batch([{k: v for k, v in u.items() if k != "spk_embed"} for u in us], spk_id=True)
    assert "spk_embed" not in pb.t
    assert pb.spk_ids.dtype == np.int32 and pb.spk_ids.tolist() == [3, 13, 23]
    for k in ("txt_tokens", "note", "note_type", "note_dur", "mel2ph", "emo_embed", "ref_mels", "ref_f0"):
        assert torch.equal(pb.t[k], full.t[k]), k
    moved = pb.to("cpu")
    assert moved.spk_ids is pb.spk_ids  # host ids stay on the host when the tensors move
    with pytest.raises(TypeError):
        pack_batch([dict(us[0], spk_id=1.5)], spk_id=True)


class _FakeEngine:
    device = torch.device("cpu")

    def __init__(self):
        self.calls = []

    def predict_durations(self, pb):
        self.calls.append({"dur": pb.spk_ids})
        return torch.full((int(pb.ph_offsets[-1]),), 6, dtype=torch.int32), None

    def forward(self, pb, noise=None, seed=0, skip_mel_diffusion=False, dur=None, want=(), **kw):
        self.calls.append({"t": set(pb.t), "spk": pb.spk_ids, "want": set(want), "skip": skip_mel_diffusion})
        Fs, B = int(pb.frame_offsets[-1]), pb.B
        shapes = {"mel_out": (Fs, 80), "coarse_mel": (Fs, 80), "f0_denorm": (Fs,), "decoder_inp": (Fs, 256),
                  "pitch_pred": (Fs, 2), "spk_proj": (B, 256), "emo_proj": (B, 256), "style": (Fs, 256)}
        out = {k: torch.zeros(shapes[k]) for k in want if k in shapes}
        out["mel2ph"] = pb.t["mel2ph"] if "mel2ph" in pb.t else torch.ones(Fs, dtype=torch.int32)
        return out


def test_facade_takes_speaker_ids_and_the_fft_decoder_ignores_diff_start():
    """modules.StyleSinger on a use_spk_id FFT model: spk_embed is a LongTensor [B] of ids, as the reference's forward
    receives it; the batch carries them as host ids and no speaker vectors.  The FFT decoder's mel is the output at any
    global_steps (no diff_start gate), and predicted durations see the same ids."""
    import stylesinger_b200.modules as M
    us = _utts(2)
    eng = _FakeEngine()
    m = M.StyleSinger(hparams=dict(decoder="fft", use_spk_id=True, **X), engine=eng)
    kw = dict(spk_embed=torch.tensor([3, 13]), emo_embed=torch.stack([u["emo_embed"] for u in us]),
              ref_mels=torch.stack([u["ref_mels"][:16] for u in us]), ref_f0=torch.stack([u["ref_f0"][:16] for u in us]),
              infer=True, note=torch.stack([u["note"] for u in us]), note_dur=torch.stack([u["note_dur"] for u in us]),
              note_type=torch.stack([u["note_type"] for u in us]))
    txt = torch.stack([u["txt_tokens"] for u in us])
    ret = m(txt, mel2ph=torch.stack([u["mel2ph"][:30] for u in us]), global_steps=30000, **kw)
    call = eng.calls[-1]
    assert "spk_embed" not in call["t"] and call["spk"].tolist() == [3, 13]
    assert "mel_out" in call["want"] and not call["skip"] and ret["mel_out"].shape == (2, 30, 80)
    m(txt, global_steps=30000, **kw)  # predicted durations
    assert eng.calls[-2]["dur"].tolist() == [3, 13] and eng.calls[-1]["spk"].tolist() == [3, 13]


def test_infer_reads_the_items_speaker_id():
    """StyleSingerInfer.input_to_batch / preprocess_input read inp['spk_id'] on a use_spk_id model (the line the
    reference leaves commented out), and formats.item_to_utterance carries the dataset's spk_id."""
    from stylesinger_b200 import formats
    from stylesinger_b200.infer import StyleSingerInfer
    inf = object.__new__(StyleSingerInfer)
    inf.hparams = resolve(use_spk_id=True, emo=False, style=False, **X)
    u = _utts(1)[0]
    item = {"ph_token": u["txt_tokens"].numpy(), "note": u["note"].numpy(), "note_dur": u["note_dur"].numpy(),
            "note_type": u["note_type"].numpy(), "spk_id": 42, "mel2ph": u["mel2ph"].numpy()}
    pb = inf.input_to_batch(item)
    assert pb.spk_ids.tolist() == [42] and "spk_embed" not in pb.t
    inf.hparams = resolve(emo=False, style=False)
    with pytest.raises(KeyError):
        inf.input_to_batch(item)  # a speaker-vector model needs item['spk_embed']
    ds_item = {"mel": np.zeros((30, 80), np.float32), "mel2ph": u["mel2ph"].numpy(), "f0": np.full(30, 200.0),
               "ph_token": u["txt_tokens"].numpy(), "ep_pitches": u["note"].numpy(), "ep_notedurs": u["note_dur"].numpy(),
               "ep_types": u["note_type"].numpy(), "spk_id": 7, "emo_embed": np.zeros(256, np.float32)}
    v = formats.item_to_utterance(ds_item, resolve(use_spk_id=True, **X))
    assert v["spk_id"] == 7 and "spk_embed" not in v


def _scatter_worker(rank, world, port, q):
    import os

    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from stylesinger_b200.dist import scatter_utterances
    utts = _utts(5) if rank == 0 else None
    pb, idx = scatter_utterances(utts, src=0, spk_id=True)
    q.put((rank, pb.spk_ids.tolist(), list(idx), "spk_embed" in pb.t))
    dist.destroy_process_group()


def test_scatter_carries_speaker_ids():
    """dist.scatter_utterances(..., spk_id=True): every rank receives its utterances' host ids and no speaker vectors."""
    import socket

    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_scatter_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for _, ids, idx, has_vec in res:
        assert ids == [10 * i + 3 for i in idx] and not has_vec
    assert sorted(sum((r[2] for r in res), [])) == [0, 1, 2, 3, 4]
