"""Per-utterance Philox seeds (ssb_acoustic_forward_keyed / ssb_hifigan_generate_keyed) on the GPU.

A keyed call gives utterance b the draws of a B = 1 call with seed = seeds[b].  Checked here: solo keyed against solo
legacy (bitwise, on every sampler path); the draws themselves, read back through test_gpu_philox's noise-reading schedule,
against the solo calls (bitwise) and the NumPy keyed plan (tests/keyed_plan.py); batch order (bitwise); batch against
solo at the bench's batch64 lengths; the vocoder under every grouping; the end-to-end entries and
tools/infer_dataset.py --seed-per-item; the workspace query."""
import os
import pickle
import sys

import numpy as np
import pytest
import torch

from stylesinger_b200 import synth
from stylesinger_b200.engine import AcousticModel, Vocoder, pack_batch
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG, resolve
from tests import keyed_plan as K
from tests.common import acoustic_sd, conv_hp, conv_sd, golden, hp_for, vocoder_sd
from tests.test_gpu_philox import TOL, _probe_schedule, _real_schedule

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WANT = ("mel_out", "f0_denorm", "pitch_pred")
_M = {}


def _utt(frames, idx):
    return synth.make_utterance(frames / 187.5, utt_idx=idx, ref_frames=60, frames=frames,
                                phones=max(1, min(frames, frames // 12 + 1)))


def _model(kind="diffsinger", T=8):
    key = (kind, T)
    if key not in _M:
        if kind == "prodiff":
            _, meta = golden("ref_prodiff_T8")
            hp = resolve(timesteps=T, K_step=T, f0_timesteps=4, **meta["overrides"])
            _M[key] = AcousticModel(synth.acoustic_state_dict(hp, seed=0), hp)
        elif kind == "conv":
            _, meta = golden("ref_convf0")
            _M[key] = AcousticModel(conv_sd(meta), conv_hp(meta))
        else:
            # positions for the 6300-frame utterance of test_keyed_draws_are_the_solo_draws_and_the_plan
            _M[key] = AcousticModel(acoustic_sd(), hp_for(T, T), max_positions=8192)
    m = _M[key]
    m.set_tensor_cores(True)
    m.set_persistent(True)
    m.set_persistent_groups(False)
    return m


def _voc():
    if "voc" not in _M:
        _M["voc"] = Vocoder(vocoder_sd(), DEFAULT_VOCODER_CONFIG)
    v = _M["voc"]
    v.set_tensor_cores(True)
    return v


def _run(m, utts, seeds=None, seed=0, want=WANT):
    """Forward of `utts` as one batch, split per utterance (numpy)."""
    pb = pack_batch(utts).to(DEV)
    out = m.forward(pb, seed=seed, seeds=seeds, want=want)
    fo = pb.frame_offsets
    return [{k: v[fo[b]:fo[b + 1]].cpu().numpy() for k, v in out.items()} for b in range(pb.B)]


def _same(a, b, what):
    for k in a:
        assert np.array_equal(a[k], b[k]), f"{what}: {k} differs, max |d| {np.abs(a[k] - b[k]).max():.3e}"


# ---- 1. solo keyed == solo legacy, bitwise ------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["tc_persistent", "tc_per_launch", "ffma", "k_step", "plms", "prodiff", "f0_conv"])
def test_solo_keyed_equals_legacy_bitwise(case):
    kind = {"prodiff": "prodiff", "f0_conv": "conv"}.get(case, "diffsinger")
    m = _model(kind)
    u = [_utt(300, 5)]
    s = 0xC0FFEE1234567890
    hp0 = m.hp
    try:
        m.set_tensor_cores(case != "ffma")
        m.set_persistent(case in ("tc_persistent", "k_step", "prodiff", "f0_conv"))
        if case == "k_step":
            m.set_mel_k_step(5)
        if case == "plms":
            m.hp = dict(hp0, pndm_speedup=3)
        a = _run(m, u, seeds=[s])[0]
        b = _run(m, u, seed=s)[0]
    finally:
        m.hp = hp0
        if case == "k_step":
            m.set_mel_k_step(None)
    _same(a, b, case)
    v = _voc()
    mel = torch.from_numpy(a["mel_out"]).to(DEV).clamp(-6, 1.5).contiguous()
    f0 = torch.from_numpy(a["f0_denorm"]).to(DEV)
    fo = np.array([0, 300], np.int32)
    wa = v.generate(mel, f0, fo, seeds=[s]).cpu().numpy()
    wb = v.generate(mel, f0, fo, seed=s).cpu().numpy()
    assert np.array_equal(wa, wb)
    print(f"{case}: mel_out, f0_denorm, pitch_pred and wav bitwise equal")


# ---- 2. the draws are the plan -------------------------------------------------------------------------------------------
RAGGED = [1, 2, 3, 5, 17, 150, 700, 6300]  # the last one alone is 50 row tiles (> 48)


@pytest.mark.parametrize("grouped", [False, True])
def test_keyed_draws_are_the_solo_draws_and_the_plan(grouped):
    """Noise-reading schedules on both samplers (T = f0_T = 4): mel_out = denorm(mel draw), pitch_pred[:, 0] = the two F0
    nets' draws summed (z_a + z_s + 8).  Each utterance's read-back equals its solo legacy call bitwise and the keyed plan
    within test_gpu_philox's bars; the plan under wrong keys misses by >= 100x."""
    m = _model("diffsinger", 4)
    utts = [_utt(f, 40 + i) for i, f in enumerate(RAGGED)]
    seeds = [(0x9E3779B97F4A7C15 * (i + 3)) % (1 << 64) for i in range(len(utts))]
    fo = np.concatenate([[0], np.cumsum(RAGGED)])
    smin = acoustic_sd()["postdiff.spec_min"].reshape(-1)[:80].numpy().astype(np.float32)
    smax = acoustic_sd()["postdiff.spec_max"].reshape(-1)[:80].numpy().astype(np.float32)
    d = smax - smin
    worst, miss = 0.0, np.inf
    try:
        m.set_persistent_groups(grouped)
        for t_star in (None, 3, 0):
            _probe_schedule(m, 0, 4, t_star)
            _probe_schedule(m, 1, 4, t_star)
            got = _run(m, utts, seeds=seeds, want=("mel_out", "pitch_pred"))
            for b, u in enumerate(utts):
                _same(got[b], _run(m, [u], seed=seeds[b], want=("mel_out", "pitch_pred"))[0], f"utt {b} t*={t_star}")
            mel = np.concatenate([g["mel_out"] for g in got]).astype(np.float64)
            pp = np.concatenate([g["pitch_pred"][:, 0] for g in got]).astype(np.float64)
            blk = 0 if t_star is None else 4 - t_star
            for ks, bad in ((seeds, False), ([s + 1 for s in seeds], True)):
                z = K.mel_noise(ks, 4, fo, steps=[] if t_star is None else [t_star])[blk]
                want_mel = (z + np.float32(1)) / np.float32(2) * d + smin
                bar_mel = TOL * np.maximum(1, np.abs(z)) * np.abs(d) / 2 + 4 * np.finfo(np.float32).eps * (
                    np.abs(want_mel) + np.abs(smin) + np.abs(d))
                zf = [K.f0_gauss_noise(ks, net, 4, fo)[blk] for net in range(2)]
                f = [(zz + np.float32(1)) / np.float32(2) * np.float32(4) + np.float32(6) for zz in zf]
                want_pp = (f[1] / np.float32(2) + f[0] / np.float32(2)).astype(np.float64)
                bar_pp = TOL * (np.maximum(1, np.abs(zf[0])) + np.maximum(1, np.abs(zf[1]))) + 4e-6
                r = max(float((np.abs(mel - want_mel) / bar_mel).max()), float((np.abs(pp - want_pp) / bar_pp).max()))
                if bad:
                    miss = min(miss, r)
                else:
                    worst = max(worst, r)
    finally:
        m.set_persistent_groups(False)
        _real_schedule(m, 4, 4)
    print(f"grouped={grouped}: {len(RAGGED)} utterances ({int(fo[-1])} frames) bitwise equal to their solo calls; "
          f"plan max |d|/bar {worst:.3f}; wrong keys miss by {miss:.0f}x the bar")
    assert worst <= 1.0 and miss >= 100


# ---- 3. order invariance -------------------------------------------------------------------------------------------------
def test_keyed_batch_order_does_not_change_any_output():
    """The same keyed batch reversed and rotated gives every utterance the same outputs.  Bitwise with the tensor-core
    attention switched off.  With it on (the default), this batch of 26 row tiles runs the FFT decoder's and the aligner's
    attention on the wgmma kernel, whose key tiles sit on an 8-row grid of the batch layout (attention_tc.cu): an
    utterance's keys are then summed in groups that depend on its first row mod 8, i.e. on the lengths in front of it.
    That holds for the per-call seed too; there the outputs agree to fp32 rounding, checked against a bar of 1e-4."""
    from stylesinger_b200._lib import lib
    m = _model("diffsinger", 8)
    lens = [1, 2, 3, 5, 17, 150, 700, 333, 1201]
    utts = [_utt(f, 60 + i) for i, f in enumerate(lens)]
    seeds = [1000 + 7 * i for i in range(len(lens))]
    n = len(lens)
    orders = (("reversed", list(range(n))[::-1]), ("rotated", list(range(3, n)) + list(range(3))))
    try:
        for attn_tc in (0, 1):
            lib.ssb_set_attention_tensor_cores(attn_tc)
            base = _run(m, utts, seeds=seeds)
            worst = 0.0
            for name, order in orders:
                got = _run(m, [utts[i] for i in order], seeds=[seeds[i] for i in order])
                for j, i in enumerate(order):
                    if not attn_tc:
                        _same(got[j], base[i], f"{name}: utterance {i}")
                        continue
                    worst = max(worst, float(np.abs(got[j]["mel_out"].astype(np.float64) - base[i]["mel_out"]).max()))
                    assert np.array_equal(got[j]["f0_denorm"] == 0, base[i]["f0_denorm"] == 0), f"{name}: uv of {i}"
            print(f"attention tensor cores {attn_tc}: " + (f"mel max |d| {worst:.3e} (bar 1e-4)" if attn_tc else
                                                           f"{n} utterances bitwise equal in every order"))
            assert worst < 1e-4
    finally:
        lib.ssb_set_attention_tensor_cores(1)


# ---- 4. batch vs solo at the bench's batch64 lengths ---------------------------------------------------------------------
def _flips(a, b):
    """Frames whose voicing (f0_denorm == 0) differs."""
    return np.nonzero((a["f0_denorm"] == 0) != (b["f0_denorm"] == 0))[0]


def _coarse(hz):
    """f0_to_coarse of the pitch embedding's input (utils/pitch_utils.py:22-31), in float64."""
    lo, hi = 1127 * np.log(1 + 50 / 700), 1127 * np.log(1 + 1100 / 700)
    mel = 1127 * np.log(1 + np.asarray(hz, np.float64) / 700)
    mel = np.where(mel > 0, (mel - lo) * 254 / (hi - lo) + 1, mel)
    return np.rint(np.clip(mel, 1, 255))


def test_keyed_batch64_equals_solo_calls():
    """T = 100, the 64 utterance lengths of bench.py --workload batch64, 8 of them compared with their solo calls:
    bitwise with FFMA forced on both sides; on the default paths within the project's T = 100 mel bar (1e-3)."""
    m = _model("diffsinger", 100)
    secs = synth.batch_seconds(64, seed=1234)
    utts = [synth.make_utterance(float(s), utt_idx=i) for i, s in enumerate(secs)]
    lens = [len(u["mel2ph"]) for u in utts]
    seeds = [(i * 0x2545F4914F6CDD1D + 17) % (1 << 64) for i in range(64)]
    pick = sorted({int(np.argmin(lens)), int(np.argmax(lens)), 0, 63, 9, 22, 37, 50})
    assert len(pick) == 8
    try:
        for ffma in (True, False):
            m.set_tensor_cores(not ffma)
            m.set_persistent(not ffma)
            batch = _run(m, utts, seeds=seeds)
            worst = 0.0
            for b in pick:
                solo = _run(m, [utts[b]], seed=seeds[b])[0]
                if ffma:
                    _same(batch[b], solo, f"FFMA, utterance {b} ({lens[b]} frames)")
                    continue
                e = float(np.abs(batch[b]["mel_out"].astype(np.float64) - solo["mel_out"]).max())
                worst = max(worst, e)
                fl = _flips(batch[b], solo)
                cb = np.nonzero(_coarse(batch[b]["f0_denorm"]) != _coarse(solo["f0_denorm"]))[0]
                for r in fl:
                    print(f"  utterance {b} frame {r}: uv flip, pitch_pred uv (batch, solo) = "
                          f"({batch[b]['pitch_pred'][r, 1]:.6g}, {solo['pitch_pred'][r, 1]:.6g})")
                for r in cb:
                    print(f"  utterance {b} frame {r}: coarse bin flip, f0_denorm (batch, solo) = "
                          f"({batch[b]['f0_denorm'][r]:.7g}, {solo['f0_denorm'][r]:.7g})")
                print(f"  utterance {b} ({lens[b]} frames): mel max |d| {e:.3e}, {len(fl)} uv flips, "
                      f"{len(cb)} coarse-bin flips")
            print(f"ffma={ffma}: " + ("8 utterances bitwise equal to their solo calls" if ffma else
                                      f"mel max |d| {worst:.3e} over 8 utterances (bar 1e-3)"))
            assert worst < 1e-3
    finally:
        m.set_tensor_cores(True)
        m.set_persistent(True)


# ---- 5. vocoder ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tc", [False, True])
def test_keyed_vocoder_batch_equals_solo_under_every_grouping(tc):
    v = _voc()
    lens = [40, 17, 25, 60, 33]
    fo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    n = int(fo[-1])
    gen = torch.Generator().manual_seed(5)
    mel = (-3.0 + 0.8 * torch.randn(n, 80, generator=gen)).clamp(-6, 1.5).to(DEV)
    f0 = 150 + 350 * torch.rand(n, generator=gen)
    f0[10:14] = 0
    f0 = f0.to(DEV)
    seeds = [77, 2**64 - 2, 0, 77, 123456789]
    mx = v.max_frames_per_call
    try:
        v.set_tensor_cores(tc)
        wavs = {}
        for cap, groups in ((mx, 1), (100, 2), (1, 5)):
            v.max_frames_per_call = cap
            wavs[groups] = v.generate(mel, f0, fo, seeds=seeds).cpu().numpy()
        v.max_frames_per_call = mx
        for b in range(len(lens)):
            a, e = int(fo[b]), int(fo[b + 1])
            solo = v.generate(mel[a:e], f0[a:e], np.array([0, e - a], np.int32), seed=seeds[b]).cpu().numpy()
            assert np.array_equal(wavs[1][a * v.hop:e * v.hop], solo), f"utterance {b}"
    finally:
        v.max_frames_per_call = mx
        v.set_tensor_cores(True)
    assert np.array_equal(wavs[1], wavs[2]) and np.array_equal(wavs[1], wavs[5])
    print(f"vocoder tc={tc}: batch = solo bitwise; 1, 2 and 5 groups bitwise equal")


# ---- 6. end to end ----------------------------------------------------------------------------------------------------
def _items(n):
    rng = np.random.default_rng(3)
    out = []
    for i in range(n):
        Fr, Pn = 50 + 23 * i, 4 + i
        f0 = rng.uniform(150, 400, Fr).astype(np.float32)
        f0[rng.random(Fr) < 0.2] = 0.0
        out.append({"item_name": f"utt{i}", "mel": np.clip(rng.normal(-3, 0.8, (Fr, 80)), -6, 0.6).astype(np.float32),
                    "f0": f0, "mel2ph": np.repeat(np.arange(1, Pn + 1), Fr // Pn + 1)[:Fr],
                    "ph_token": rng.integers(3, 60, Pn), "ep_pitches": rng.integers(48, 72, Pn),
                    "ep_notedurs": rng.uniform(0.1, 0.6, Pn), "ep_types": rng.integers(1, 3, Pn),
                    "spk_embed": rng.normal(size=256).astype(np.float32),
                    "emo_embed": rng.normal(size=256).astype(np.float32)})
    return out


def _wav_bar(a, b, what):
    e = float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())
    print(f"  {what}: wav max |d| {e:.3e}")
    return e


def test_end_to_end_keyed_batch_and_seed_per_item(tmp_path):
    """StyleSingerInfer.infer_batch(utts, seeds) against forward_model(item, seed); tools/infer_dataset.py
    --seed-per-item at --batch 64 and 5 against forward_model.  T = 8, ground-truth durations."""
    import yaml
    from scipy.io import wavfile

    from stylesinger_b200 import formats
    from stylesinger_b200.infer import StyleSingerInfer
    T = 8
    hp = resolve(timesteps=T, K_step=T, f0_timesteps=T)
    sd, vsd = synth.acoustic_state_dict(hp, seed=0), synth.vocoder_state_dict(DEFAULT_VOCODER_CONFIG, seed=0)
    eng = StyleSingerInfer(hp, DEV, sd, vsd, DEFAULT_VOCODER_CONFIG)
    items = _items(7)
    seeds = [40 + i for i in range(len(items))]
    utts = [formats.item_to_utterance(it, hp, with_mel2ph=True) for it in items]
    batch = eng.infer_batch(utts, seeds=seeds, use_mel2ph=True)
    # the same utterance in forward_model's input format (inference/StyleSinger.py's item)
    solo = [eng.forward_model({"ph_token": it["ph_token"], "note": it["ep_pitches"], "note_dur": it["ep_notedurs"],
                               "note_type": it["ep_types"], "spk_embed": it["spk_embed"], "emo_embed": it["emo_embed"],
                               "mel": it["mel"], "f0": it["f0"], "mel2ph": it["mel2ph"]}, seed=s)
            for it, s in zip(items, seeds)]
    worst = max(_wav_bar(a, b, f"infer_batch item {i}") for i, (a, b) in enumerate(zip(batch, solo)))
    assert all(len(a) == len(b) for a, b in zip(batch, solo))
    exp, voc, data = (str(tmp_path / d) for d in ("exp", "hifigan", "binary"))
    for d in (exp, voc, data):
        os.makedirs(d)
    torch.save({"state_dict": {"model": sd}}, os.path.join(exp, "model_ckpt_steps_100.ckpt"))
    torch.save({"state_dict": {"model_gen": vsd}}, os.path.join(voc, "model_ckpt_steps_1.ckpt"))
    yaml.safe_dump(dict(DEFAULT_VOCODER_CONFIG), open(os.path.join(voc, "config.yaml"), "w"))
    prefix = os.path.join(data, "test")
    offs = [0]
    with open(prefix + ".data", "wb") as f:
        for it in items:
            offs.append(offs[-1] + f.write(pickle.dumps(it)))
    np.save(open(prefix + ".idx", "wb"), {"offsets": offs})
    sys.path.insert(0, os.path.join(REPO, "tools"))
    import infer_dataset
    got = {}
    for bs in (64, 5):
        out = str(tmp_path / f"out{bs}")
        sys.argv = ["infer_dataset.py", "--ckpt", exp, "--vocoder", voc, "--data", prefix, "--out", out, "--batch",
                    str(bs), "--T", str(T), "--use-gt-dur", "--seed", "40", "--seed-per-item"]
        infer_dataset.main()
        got[bs] = [wavfile.read(os.path.join(out, f"utt{i}.wav"))[1] for i in range(len(items))]
    for bs in (64, 5):
        for i in range(len(items)):
            worst = max(worst, _wav_bar(got[bs][i], solo[i], f"--batch {bs} item {i}"))
    print(f"end to end: wav max |d| {worst:.3e} against forward_model")
    assert worst < 1e-3


# ---- 7. workspace ----------------------------------------------------------------------------------------------------------
def test_keyed_calls_run_in_the_legacy_workspace_query():
    import ctypes as C

    from stylesinger_b200._lib import AcousticOutputs, lib
    m = _model("diffsinger", 8)
    utts = [_utt(f, 80 + i) for i, f in enumerate([90, 7, 300])]
    pb = pack_batch(utts).to(DEV)
    a = m._inputs(pb)
    n = lib.ssb_acoustic_workspace_bytes(m._h, C.byref(a))
    assert n > 0
    F = int(pb.frame_offsets[-1])
    mel = torch.empty(F, 80, device=DEV)
    o = AcousticOutputs()
    o.mel_out = mel.data_ptr()
    ws = torch.empty(n, dtype=torch.uint8, device=DEV)
    keys = np.array([5, 6, 7], np.uint64)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.ssb_acoustic_forward_keyed(m._h, C.byref(a), keys.ctypes.data, C.byref(o), ws.data_ptr(), n, stream) == 0
    torch.cuda.synchronize()
    v = _voc()
    fo = np.array([0, 90, 97, 397], np.int32)
    nv = lib.ssb_vocoder_workspace_bytes(v._h, fo.ctypes.data, 3)
    wsv = torch.empty(nv, dtype=torch.uint8, device=DEV)
    wav = torch.empty(F * v.hop, device=DEV)
    f0 = torch.full((F,), 200.0, device=DEV)
    rc = lib.ssb_hifigan_generate_keyed(v._h, mel.data_ptr(), f0.data_ptr(), fo.ctypes.data, 3, keys.ctypes.data,
                                        wav.data_ptr(), wsv.data_ptr(), nv, stream)
    torch.cuda.synchronize()
    assert rc == 0 and torch.isfinite(wav).all()
    # NULL seeds and injected noise are refused by the C entries themselves
    assert lib.ssb_acoustic_forward_keyed(m._h, C.byref(a), None, C.byref(o), ws.data_ptr(), n, stream) != 0
    a.mel_noise = mel.data_ptr()
    assert lib.ssb_acoustic_forward_keyed(m._h, C.byref(a), keys.ctypes.data, C.byref(o), ws.data_ptr(), n, stream) != 0
    assert lib.ssb_hifigan_generate_keyed(v._h, mel.data_ptr(), f0.data_ptr(), fo.ctypes.data, 3, None,
                                          wav.data_ptr(), wsv.data_ptr(), nv, stream) != 0
    print(f"keyed forward in {n} bytes, keyed vocoder in {nv} bytes: the legacy queries' sizes")
