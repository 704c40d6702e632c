"""Generate tests/golden/*.npz by executing the UNMODIFIED reference (build container only).

    python tools/make_golden.py            # writes tests/golden/

What it does (SURVEY.md §8c): imports /root/reference through tools/ref_import.py, builds the
reference's own ``StyleSinger`` / ``HifiGanGenerator`` modules, loads the synthetic checkpoints of
``stylesinger_b200.synth`` with ``strict=True`` (which also proves state-dict name/shape
compatibility with released checkpoints), monkey-patches ``torch.randn/randn_like/rand/rand_like``
to a seeded ``NoiseSource`` so the stochastic samplers are reproducible, runs the reference and
dumps small fixtures.  The fixtures pin oracle/stylesinger_oracle.py (tests/test_oracle_golden.py)
and, through it and directly, the CUDA path (tests/test_gpu_*.py).
"""
import contextlib
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

from oracle.stylesinger_oracle import NoiseSource  # noqa: E402
from stylesinger_b200 import synth  # noqa: E402
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG  # noqa: E402
from tests.common import registry_inputs  # noqa: E402

OUT = os.path.join(REPO, "tests", "golden")


@contextlib.contextmanager
def patched_rng(ns):
    o = (torch.randn, torch.randn_like, torch.rand, torch.rand_like)

    def _shape(a):
        if len(a) == 1 and isinstance(a[0], (tuple, list, torch.Size)):
            return tuple(a[0])
        return tuple(a)

    torch.randn = lambda *a, **k: ns.randn(_shape(a))
    torch.randn_like = lambda x, **k: ns.randn(tuple(x.shape))
    torch.rand = lambda *a, **k: ns.rand(_shape(a))
    torch.rand_like = lambda x, **k: ns.rand(tuple(x.shape))
    try:
        yield
    finally:
        torch.randn, torch.randn_like, torch.rand, torch.rand_like = o


class _Dict:
    def pad(self):
        return 0

    def __len__(self):
        return synth.N_TOKENS


def build_reference_model(T, f0_T=None, K=None):
    import ref_import
    hp = ref_import.install(T=T, f0_T=f0_T)
    if K is not None:  # StyleSinger.__init__ hands hparams['K_step'] to the DiffusionDecoder (stylesinger.py:103-110)
        hp["K_step"] = K
    # fresh import state for every T: the schedule buffers are built in __init__
    import modules.diff.shallow_diffusion_tts as sdt
    import modules.diff.gaussian_multinomial_diffusion as gmd
    sdt.tqdm = lambda it, **k: it
    gmd.tqdm = lambda it, **k: it
    from modules.StyleSinger.stylesinger import StyleSinger
    model = StyleSinger(_Dict()).eval()
    sd = synth.acoustic_state_dict(dict(hp, K_step=T), seed=0)  # the weights do not depend on K_step
    missing, unexpected = model.load_state_dict(sd, strict=True), None
    return model, hp, sd


def batchify(u):
    return dict(txt_tokens=u["txt_tokens"][None], note=u["note"][None], note_dur=u["note_dur"][None],
                note_type=u["note_type"][None], spk_embed=u["spk_embed"][None], emo_embed=u["emo_embed"][None],
                ref_mels=u["ref_mels"][None], ref_f0=u["ref_f0"])  # ref_f0 is 1-D at B=1 (inference/StyleSinger.py:151)


def run_model(model, u, seed, mel2ph=True, global_steps=320000):
    ns = NoiseSource(seed)
    b = batchify(u)
    cap = {}
    h = model.style_extractor.rqvae.register_forward_hook(lambda m, i, o: cap.__setitem__("rq_in", i[0].detach().clone()))
    with torch.no_grad(), patched_rng(ns):
        out = model(b["txt_tokens"], mel2ph=u["mel2ph"][None] if mel2ph else None, spk_embed=b["spk_embed"],
                    emo_embed=b["emo_embed"], ref_mels=b["ref_mels"].clone(), ref_f0=b["ref_f0"].clone(),
                    global_steps=global_steps, infer=True, note=b["note"], note_dur=b["note_dur"],
                    note_type=b["note_type"])
        codes = model.style_extractor.rqvae.quantize(cap["rq_in"])[1]
    h.remove()
    out["rq_codes"] = codes
    out["rq_in"] = cap["rq_in"]
    return out, ns.log


def np32(t):
    return t.detach().cpu().numpy().astype(np.float32)


def case_model(name, T, frames, phones, ref_frames, seed, utt_idx, with_dur_case=True):
    model, hp, sd = build_reference_model(T)
    u = synth.make_utterance(frames / 187.5, utt_idx=utt_idx, ref_frames=ref_frames, frames=frames, phones=phones)
    out, log = run_model(model, u, seed)
    coarse, _ = run_model(model, u, seed, global_steps=50000)  # forcing < global_steps < diff_start: coarse mel only
    d = {
        "meta": json.dumps({"T": T, "frames": frames, "phones": phones, "ref_frames": ref_frames, "seed": seed,
                            "utt_idx": utt_idx, "noise_log": log}),
        "style": np32(out["style"][0]), "rq_codes": out["rq_codes"][0].numpy().astype(np.int64),
        "rq_in": np32(out["rq_in"][0]),
        "pitch_pred": np32(out["pitch_pred"][0]), "f0_denorm": np32(out["f0_denorm"][0]),
        "decoder_inp": np32(out["decoder_inp"][0]), "coarse_mel": np32(coarse["mel_out"][0]),
        "mel_out": np32(out["mel_out"][0]), "spk_embed": np32(out["spk_embed"][0]), "emo_embed": np32(out["emo_embed"][0]),
    }
    if with_dur_case:
        o2, log2 = run_model(model, u, seed + 1, mel2ph=False)
        d.update({"dur_mel2ph": o2["mel2ph"][0].numpy().astype(np.int64), "dur_logdur": np32(o2["dur"][0]),
                  "dur_mel_out": np32(o2["mel_out"][0]), "dur_f0_denorm": np32(o2["f0_denorm"][0]),
                  "dur_noise_log": json.dumps(log2)})
    # single denoiser evaluations (deterministic)
    g = torch.Generator().manual_seed(99)
    Fr = 48
    spec = torch.randn(1, 1, 80, Fr, generator=g)
    cond = torch.randn(1, 256, Fr, generator=g)
    with torch.no_grad():
        e1 = model.postdiff.denoise_fn(spec, torch.tensor([T - 1]), cond)
        f0 = torch.randn(1, 1, Fr, generator=g)
        uv = (torch.rand(1, Fr, generator=g) < 0.4).long()
        e2 = model.gm_diffnet(f0, uv, torch.tensor([1]), cond, torch.ones(1, Fr))
        e3 = model.gm_diffnet_inpainte(f0, uv, torch.tensor([0]), cond, torch.ones(1, Fr))
    d.update({"dn_spec": np32(spec[0, 0]), "dn_cond": np32(cond[0]), "dn_out": np32(e1[0, 0]),
              "dd_f0": np32(f0[0, 0]), "dd_uv": uv[0].numpy().astype(np.int64), "dd_out": np32(e2[0]),
              "dd_out_inp": np32(e3[0])})
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, {k: (v.shape if hasattr(v, "shape") else "meta") for k, v in d.items()})


def padded_utterance(frames, phones, ref_frames, utt_idx, pad_phones=3, gap=(52, 60), tail_frames=10,
                     ref_tail=8, ref_col0_row=17):
    """A synthetic utterance with every kind of padding the model masks: `pad_phones` trailing padding phones (token,
    note, note_type and note_dur 0), an interior run `gap` and a trailing run of padding frames (mel2ph 0), `ref_tail`
    all-zero reference-mel rows at the end (ref_f0 0 there) and one interior reference row whose column 0 alone is 0
    (column-0 masks drop it, whole-row masks keep it)."""
    u = synth.make_utterance(frames / 187.5, utt_idx=utt_idx, ref_frames=ref_frames, frames=frames, phones=phones)
    for k in ("txt_tokens", "note", "note_type", "note_dur"):
        u[k] = torch.cat([u[k], torch.zeros(pad_phones, dtype=u[k].dtype)])
    u["mel2ph"][gap[0]:gap[1]] = 0
    u["mel2ph"][frames - tail_frames:] = 0
    u["ref_mels"][ref_frames - ref_tail:] = 0
    u["ref_f0"][ref_frames - ref_tail:] = 0
    u["ref_mels"][ref_col0_row, 0] = 0
    return u


UTT_KEYS = ("txt_tokens", "note", "note_dur", "note_type", "mel2ph", "spk_embed", "emo_embed", "ref_mels", "ref_f0")


def case_padded(name, T=4, frames=120, phones=12, ref_frames=48, seed=91, utt_idx=104):
    """Padding phones, padding frames (interior and trailing) and a padded reference mel through the full forward, with
    mel2ph given and through the duration path.  The inputs are stored in the fixture (in_*): they are not what
    synth.make_utterance returns."""
    model, hp, sd = build_reference_model(T)
    u = padded_utterance(frames, phones, ref_frames, utt_idx)
    out, log = run_model(model, u, seed)
    coarse, _ = run_model(model, u, seed, global_steps=50000)
    o2, log2 = run_model(model, u, seed + 1, mel2ph=False)
    d = {
        "meta": json.dumps({"T": T, "frames": frames, "phones": phones, "ref_frames": ref_frames, "seed": seed,
                            "utt_idx": utt_idx, "noise_log": log, "dur_noise_log": log2}),
        "style": np32(out["style"][0]), "rq_codes": out["rq_codes"][0].numpy().astype(np.int64),
        "rq_in": np32(out["rq_in"][0]),
        "pitch_pred": np32(out["pitch_pred"][0]), "f0_denorm": np32(out["f0_denorm"][0]),
        "decoder_inp": np32(out["decoder_inp"][0]), "coarse_mel": np32(coarse["mel_out"][0]),
        "mel_out": np32(out["mel_out"][0]),
        "dur_mel2ph": o2["mel2ph"][0].numpy().astype(np.int64), "dur_logdur": np32(o2["dur"][0]),
        "dur_mel_out": np32(o2["mel_out"][0]), "dur_f0_denorm": np32(o2["f0_denorm"][0]),
    }
    for k in UTT_KEYS:
        d["in_" + k] = u[k].numpy()
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, {k: (v.shape if hasattr(v, "shape") else "meta") for k, v in d.items()})


def case_vocoder(name, frames, seed):
    import ref_import
    ref_import.install(T=4)
    from modules.hifigan.hifigan_nsf import HifiGanGenerator
    h = dict(DEFAULT_VOCODER_CONFIG)
    vsd = synth.vocoder_state_dict(h, seed=0)
    gen = HifiGanGenerator(h)
    gen.load_state_dict(vsd, strict=True)
    gen.remove_weight_norm()
    gen.eval()
    g = torch.Generator().manual_seed(seed)
    mel = (-3.0 + 0.8 * torch.randn(frames, 80, generator=g)).clamp(-6, 1.5)
    f0 = 150 + 350 * torch.rand(frames, generator=g)
    f0[frames // 3: frames // 3 + 5] = 0  # an unvoiced stretch
    ns = NoiseSource(seed + 5)
    with torch.no_grad(), patched_rng(ns):
        c = torch.FloatTensor(mel.numpy()).unsqueeze(0).transpose(2, 1)
        y = gen(c, torch.FloatTensor(f0.numpy()[None, :])).view(-1)
        ns2 = NoiseSource(seed + 6)
    with torch.no_grad():
        y_nof0 = gen(c).view(-1)
    d = {"meta": json.dumps({"frames": frames, "seed": seed, "noise_log": ns.log}), "mel": np32(mel), "f0": np32(f0),
         "wav": np32(y), "wav_nof0": np32(y_nof0)}
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, y.shape, float(y.abs().max()), float(y.std()))


VOCODER_EDGE_LENGTHS = (1, 2, 3, 5, 17)


def case_vocoder_edges(name, lengths=VOCODER_EDGE_LENGTHS, seed=37):
    """The reference HifiGanGenerator (B = 1) on utterances shorter than conv_pre's reach of 3 frames and just past a
    16-frame tile, with and without f0.  f0 alternates voiced / unvoiced every frame; the 5- and 17-frame utterances
    carry one frame at ~1100 Hz (9 harmonics up to ~9.9 kHz) and the 3-frame one is entirely unvoiced.  Every mel holds
    values at both clip bounds (-6 and 1.5).  The inputs are stored (mel_<L>, f0_<L>); the noise of length L is drawn from
    NoiseSource(seed + L), logged in meta."""
    import ref_import
    ref_import.install(T=4)
    from modules.hifigan.hifigan_nsf import HifiGanGenerator
    h = dict(DEFAULT_VOCODER_CONFIG)
    gen = HifiGanGenerator(h)
    gen.load_state_dict(synth.vocoder_state_dict(h, seed=0), strict=True)
    gen.remove_weight_norm()
    gen.eval()
    g = torch.Generator().manual_seed(seed)
    d, logs = {}, {}
    for L in lengths:
        mel = (-3.0 + 2.0 * torch.randn(L, 80, generator=g)).clamp(-6, 1.5)
        mel[:, 0], mel[:, 79] = -6.0, 1.5
        f0 = 150 + 350 * torch.rand(L, generator=g)
        f0[1::2] = 0
        if L == 3:
            f0[:] = 0
        if L in (5, 17):
            f0[2] = 1100.0
        ns = NoiseSource(seed + L)
        with torch.no_grad(), patched_rng(ns):
            c = mel.t()[None].contiguous()
            y = gen(c, f0[None].clone()).view(-1)
        with torch.no_grad():
            y_nof0 = gen(c).view(-1)
        logs[L] = ns.log
        d.update({f"mel_{L}": np32(mel), f"f0_{L}": np32(f0), f"wav_{L}": np32(y), f"wav_nof0_{L}": np32(y_nof0)})
    d["meta"] = json.dumps({"lengths": list(lengths), "seed": seed, "noise_log": {str(k): v for k, v in logs.items()}})
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, {k: v.shape for k, v in d.items() if k != "meta"})


VOCODER_LAYOUT_LENGTHS = (1, 2, 3, 5, 17, 24)


def case_vocoder_layouts(name, lengths=VOCODER_LAYOUT_LENGTHS, seed=53):
    """The reference HifiGanGenerator (B = 1) in HiFi-GAN's other two published layouts: V2 (ResBlock1, stages of 64,
    32, 16 and 8 channels), V3 (ResBlock2 over stages of 128, 64 and 32 channels) and V3 without the NSF source (the
    generator of a config with use_pitch_embed: False, run without f0).  Synthetic weights from synth.vocoder_state_dict,
    loaded with strict=True, weight norm removed.  One mel / f0 pair per length (stored as mel_<L>, f0_<L>), shared by
    the layouts; f0 has an unvoiced frame every third frame.  The noise of length L is NoiseSource(seed + L), as in
    case_vocoder_edges.  The reference's state-dict keys (weight-norm form) are stored per layout in meta."""
    import ref_import
    ref_import.install(T=4)
    from modules.hifigan.hifigan_nsf import HifiGanGenerator
    from stylesinger_b200.hparams import HIFIGAN_V2, HIFIGAN_V3
    layouts = {"v2": HIFIGAN_V2, "v3": HIFIGAN_V3, "v3_nonsf": dict(HIFIGAN_V3, use_pitch_embed=False)}
    g = torch.Generator().manual_seed(seed)
    d, keys = {}, {}
    inputs = {}
    for L in lengths:
        mel = (-3.0 + 1.0 * torch.randn(L, 80, generator=g)).clamp(-6, 1.5)
        f0 = 150 + 350 * torch.rand(L, generator=g)
        f0[1::3] = 0
        inputs[L] = (mel, f0)
        d.update({f"mel_{L}": np32(mel), f"f0_{L}": np32(f0)})
    for lname, h in layouts.items():
        gen = HifiGanGenerator(h)
        keys[lname] = list(gen.state_dict().keys())
        gen.load_state_dict(synth.vocoder_state_dict(h, seed=0), strict=True)
        gen.remove_weight_norm()
        gen.eval()
        for L in lengths:
            mel, f0 = inputs[L]
            c = mel.t()[None].contiguous()
            if h["use_pitch_embed"]:
                ns = NoiseSource(seed + L)
                with torch.no_grad(), patched_rng(ns):
                    y = gen(c, f0[None].clone()).view(-1)
                d[f"wav_{lname}_{L}"] = np32(y)
                print(f"{lname} L={L:2d} f0:    max |wav| {float(y.abs().max()):.3f} std {float(y.std()):.3f}")
            with torch.no_grad():
                y = gen(c).view(-1)
            d[f"wav_nof0_{lname}_{L}"] = np32(y)
            print(f"{lname} L={L:2d} no f0: max |wav| {float(y.abs().max()):.3f} std {float(y.std()):.3f}")
    d["meta"] = json.dumps({"lengths": list(lengths), "seed": seed, "layouts": list(layouts), "keys": keys})
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, len(d) - 1, "arrays")


def case_plms(name, T=100, interval=10, frames=48, seed=61):
    """f2: the reference's PLMS sampler (GaussianDiffusion.p_sample_plms, shallow_diffusion_tts.py:164-197) driven exactly
    as GaussianDiffusion.forward does under hparams['pndm_speedup'] (:254-260), on the StyleSinger mel denoiser (the
    DiffusionDecoder instance inherits the method)."""
    from collections import deque
    model, hp, sd = build_reference_model(T)
    pd = model.postdiff
    g = torch.Generator().manual_seed(seed)
    cond = torch.randn(1, frames, 256, generator=g)
    coarse = (-3 + 0.8 * torch.randn(1, frames, 80, generator=g)).clamp(-6, 0.5)
    ns = NoiseSource(seed + 1)
    with torch.no_grad(), patched_rng(ns):
        c = cond.transpose(1, 2)
        fs2 = pd.norm_spec(coarse).transpose(1, 2)[:, None, :, :]
        x = pd.q_sample(x_start=fs2, t=torch.tensor([T - 1]).long())
        pd.noise_list = deque(maxlen=4)
        for i in reversed(range(0, T, interval)):
            x = pd.p_sample_plms(x, torch.full((1,), i, dtype=torch.long), interval, c)
        mel = pd.denorm_spec(x[:, 0].transpose(1, 2))
    d = {"meta": json.dumps({"T": T, "interval": interval, "frames": frames, "seed": seed, "noise_log": ns.log}),
         "cond": np32(cond[0]), "coarse": np32(coarse[0]), "mel": np32(mel[0])}
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, mel.shape, float(mel.abs().max()))


def case_kstep(name, T_fwd=25, K_fwd=11, frames=64, phones=8, ref_frames=48, seed=141, utt_idx=106, T=100, K=51,
               intervals=(10, 7), sampler_frames=48):
    """Shallow diffusion, hparams['K_step'] < timesteps (GaussianDiffusion.__init__ :92, DiffusionDecoder.forward :297-304):
    x_K = q_sample(norm_spec(coarse), K - 1) on the T-step schedule, then K reverse steps.
    (a) fwd_*: a full B = 1 forward at T_fwd / K_fwd with mel2ph given, and its coarse mel;
    (b) smp_*: DiffusionDecoder.forward(infer=True) alone at T / K on seeded cond and coarse;
    (c) plms_i<k>_*: the PLMS loop driven as case_plms does but from t = K (t0 = the largest multiple of k below K);
    (d) smp1_*: (b) at K = 1, one step at t = 0 (its noise is drawn and multiplied by 0).
    Every noise log is in meta."""
    from collections import deque
    model, hp, sd = build_reference_model(T_fwd, K=K_fwd)
    assert model.postdiff.K_step == K_fwd and model.postdiff.num_timesteps == T_fwd
    u = synth.make_utterance(frames / 187.5, utt_idx=utt_idx, ref_frames=ref_frames, frames=frames, phones=phones)
    out, log = run_model(model, u, seed)
    coarse_fwd, _ = run_model(model, u, seed, global_steps=50000)  # forcing < global_steps < diff_start: coarse mel only
    meta = {"T_fwd": T_fwd, "K_fwd": K_fwd, "frames": frames, "phones": phones, "ref_frames": ref_frames, "seed": seed,
            "utt_idx": utt_idx, "noise_log": log, "T": T, "K": K, "intervals": list(intervals),
            "sampler_frames": sampler_frames}
    d = {"fwd_style": np32(out["style"][0]), "fwd_rq_codes": out["rq_codes"][0].numpy().astype(np.int64),
         "fwd_pitch_pred": np32(out["pitch_pred"][0]), "fwd_f0_denorm": np32(out["f0_denorm"][0]),
         "fwd_decoder_inp": np32(out["decoder_inp"][0]), "fwd_coarse_mel": np32(coarse_fwd["mel_out"][0]),
         "fwd_mel_out": np32(out["mel_out"][0])}
    g = torch.Generator().manual_seed(seed + 1)
    cond = torch.randn(1, sampler_frames, 256, generator=g)
    coarse = (-3 + 0.8 * torch.randn(1, sampler_frames, 80, generator=g)).clamp(-6, 0.5)
    d.update({"smp_cond": np32(cond[0]), "smp_coarse": np32(coarse[0])})
    for key, k_step in (("smp", K), ("smp1", 1)):
        model, _, _ = build_reference_model(T, K=k_step)
        pd = model.postdiff
        assert pd.K_step == k_step and pd.num_timesteps == T
        ns = NoiseSource(seed + 2)
        ret = {}
        with torch.no_grad(), patched_rng(ns):
            pd(cond, None, coarse, ret, infer=True)
        d[key + "_mel"] = np32(ret["mel_out"][0])
        meta[key + "_noise_log"] = ns.log
    model, _, _ = build_reference_model(T, K=K)
    pd = model.postdiff
    for k in intervals:
        ns = NoiseSource(seed + 3)
        with torch.no_grad(), patched_rng(ns):
            c = cond.transpose(1, 2)
            fs2 = pd.norm_spec(coarse).transpose(1, 2)[:, None, :, :]
            t = pd.K_step
            x = pd.q_sample(x_start=fs2, t=torch.tensor([t - 1]).long())
            pd.noise_list = deque(maxlen=4)
            steps = list(reversed(range(0, t, k)))
            for i in steps:
                x = pd.p_sample_plms(x, torch.full((1,), i, dtype=torch.long), k, c)
            mel = pd.denorm_spec(x[:, 0].transpose(1, 2))
        d[f"plms_i{k}_mel"] = np32(mel[0])
        meta[f"plms_i{k}_noise_log"] = ns.log
        meta[f"plms_i{k}_t0"] = steps[0]
    d["meta"] = json.dumps(meta)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, {k: (v.shape if hasattr(v, "shape") else "meta") for k, v in d.items()},
          {k: v for k, v in meta.items() if k.endswith("_t0")})


PRODIFF_OVERRIDES = {"decoder": "prodiff", "schedule_type": "vpsde", "timescale": 1}  # egs/stylesinger.yaml:145-155


def case_prodiff(name, T=8, f0_T=4, frames=32, phones=4, ref_frames=32, seed=81, utt_idx=103, sampler_frames=48):
    """The ProDiff teacher mel decoder (hparams['decoder'] == 'prodiff', stylesinger.py:111-117,176-177,
    modules/diff/prodiff.py:59-232) with the vpsde schedule: a full B=1 forward, a sampler-only run of
    ProDiffusion.forward(cond, infer=True) on seeded cond, the registered schedule buffers and the state dict's key list."""
    import ref_import
    hp = ref_import.install(T=T, f0_T=f0_T, overrides=PRODIFF_OVERRIDES)
    import modules.diff.prodiff as pdm
    import modules.diff.gaussian_multinomial_diffusion as gmd
    pdm.tqdm = lambda it, **k: it
    gmd.tqdm = lambda it, **k: it
    from modules.StyleSinger.stylesinger import StyleSinger
    model = StyleSinger(_Dict()).eval()
    sd = synth.acoustic_state_dict(dict(hp), seed=0)
    model.load_state_dict(sd, strict=True)
    u = synth.make_utterance(frames / 187.5, utt_idx=utt_idx, ref_frames=ref_frames, frames=frames, phones=phones)
    out, log = run_model(model, u, seed)
    g = torch.Generator().manual_seed(seed + 2)
    cond = torch.randn(1, sampler_frames, 256, generator=g)
    ns = NoiseSource(seed + 3)
    with torch.no_grad(), patched_rng(ns):
        smp = model.diff_decoder(cond, infer=True)["mel_out"]
    gk = ["betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod",
          "log_one_minus_alphas_cumprod", "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_variance",
          "posterior_log_variance_clipped", "posterior_mean_coef1", "posterior_mean_coef2"]
    keys = [[k, list(v.shape)] for k, v in model.state_dict().items()]
    d = {"meta": json.dumps({"T": T, "f0_T": f0_T, "frames": frames, "phones": phones, "ref_frames": ref_frames,
                             "seed": seed, "utt_idx": utt_idx, "noise_log": log, "sampler_frames": sampler_frames,
                             "sampler_seed": seed + 3, "sampler_noise_log": ns.log, "overrides": PRODIFF_OVERRIDES,
                             "state_dict": keys}),
         "mel_out": np32(out["mel_out"][0]), "f0_denorm": np32(out["f0_denorm"][0]),
         "decoder_inp": np32(out["decoder_inp"][0]), "sampler_cond": np32(cond[0]), "sampler_mel": np32(smp[0])}
    for k in gk:
        d["sched_" + k] = np32(getattr(model.diff_decoder, k))
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, {k: (v.shape if hasattr(v, "shape") else "meta") for k, v in d.items()})


CONVF0_OVERRIDES = {"f0_gen": "conv"}
CONVF0_ZERO_ROWS = (0, 7, 150, 151, 299)  # rows of the predictor-only inputs whose channel 0 is exactly 0


def case_convf0(name, T=4, frames=96, phones=12, ref_frames=64, seed=111, utt_idx=105, pred_frames=300,
                prodiff_T=8, prodiff_frames=32, prodiff_phones=4, prodiff_seed=121, prodiff_utt_idx=106):
    """The convolutional F0 generator (hparams['f0_gen'] == 'conv', stylesinger.py:73-82,223-225: two FastSpeech-2
    PitchPredictors, tts_modules.py:191-234): a B=1 full forward with mel2ph given and with predicted durations
    (DiffSinger decoder), each predictor alone on seeded inputs whose channel 0 is exactly 0 in a few rows (the
    position skip of make_positions), a B=1 full forward with the ProDiff decoder, and both state dicts' key lists."""
    import ref_import
    hp = ref_import.install(T=T, overrides=CONVF0_OVERRIDES)
    import modules.diff.shallow_diffusion_tts as sdt
    sdt.tqdm = lambda it, **k: it
    from modules.StyleSinger.stylesinger import StyleSinger
    model = StyleSinger(_Dict()).eval()
    model.load_state_dict(synth.acoustic_state_dict(dict(hp), seed=0), strict=True)
    u = synth.make_utterance(frames / 187.5, utt_idx=utt_idx, ref_frames=ref_frames, frames=frames, phones=phones)
    out, log = run_model(model, u, seed)
    o2, log2 = run_model(model, u, seed + 1, mel2ph=False)
    g = torch.Generator().manual_seed(seed + 2)
    xs = torch.randn(2, 1, pred_frames, 256, generator=g)
    xs[:, :, list(CONVF0_ZERO_ROWS), 0] = 0
    with torch.no_grad():
        pa = model.pitch_predictor(xs[0].clone())
        ps = model.pitch_inpainter_predictor(xs[1].clone())
    keys = [[k, list(v.shape)] for k, v in model.state_dict().items()]
    d = {"pitch_pred": np32(out["pitch_pred"][0]), "f0_denorm": np32(out["f0_denorm"][0]),
         "decoder_inp": np32(out["decoder_inp"][0]), "mel_out": np32(out["mel_out"][0]),
         "dur_mel2ph": o2["mel2ph"][0].numpy().astype(np.int64), "dur_pitch_pred": np32(o2["pitch_pred"][0]),
         "dur_f0_denorm": np32(o2["f0_denorm"][0]), "dur_decoder_inp": np32(o2["decoder_inp"][0]),
         "dur_mel_out": np32(o2["mel_out"][0]),
         # the predictor inputs are regenerated from pred_seed by the tests (tests/common.predictor_inputs); their
         # first rows are kept to check that
         "pred_x_head": np32(xs[:, 0, :4]), "pred_out_agnostic": np32(pa[0]), "pred_out_specific": np32(ps[0])}
    # (d) ProDiff decoder + conv F0 generator: the fast configuration
    hp2 = ref_import.install(T=prodiff_T, overrides=dict(PRODIFF_OVERRIDES, **CONVF0_OVERRIDES))
    import modules.diff.prodiff as pdm
    pdm.tqdm = lambda it, **k: it
    model2 = StyleSinger(_Dict()).eval()
    model2.load_state_dict(synth.acoustic_state_dict(dict(hp2), seed=0), strict=True)
    u2 = synth.make_utterance(prodiff_frames / 187.5, utt_idx=prodiff_utt_idx, ref_frames=prodiff_frames,
                              frames=prodiff_frames, phones=prodiff_phones)
    out2, log3 = run_model(model2, u2, prodiff_seed)
    keys2 = [[k, list(v.shape)] for k, v in model2.state_dict().items()]
    d.update({"pd_pitch_pred": np32(out2["pitch_pred"][0]), "pd_f0_denorm": np32(out2["f0_denorm"][0]),
              "pd_decoder_inp": np32(out2["decoder_inp"][0]), "pd_mel_out": np32(out2["mel_out"][0])})
    d["meta"] = json.dumps({"T": T, "frames": frames, "phones": phones, "ref_frames": ref_frames, "seed": seed,
                            "utt_idx": utt_idx, "noise_log": log, "dur_noise_log": log2, "overrides": CONVF0_OVERRIDES,
                            "pred_frames": pred_frames, "pred_seed": seed + 2, "pred_zero_rows": list(CONVF0_ZERO_ROWS),
                            "state_dict": keys,
                            "prodiff": {"T": prodiff_T, "frames": prodiff_frames, "phones": prodiff_phones,
                                        "ref_frames": prodiff_frames, "seed": prodiff_seed, "utt_idx": prodiff_utt_idx,
                                        "noise_log": log3, "overrides": dict(PRODIFF_OVERRIDES, **CONVF0_OVERRIDES),
                                        "state_dict": keys2}})
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, {k: (v.shape if hasattr(v, "shape") else "meta") for k, v in d.items()})


# The model-switch configurations (egs/stylesinger.yaml "choices of models" + use_txt_cond): name -> hparams overrides
_OFF4 = {"emo": False, "style": False, "umln": False, "use_txt_cond": False}
SWITCH_CONFIGS = {
    "no_emo": {"emo": False},
    "no_style": {"style": False},
    "no_umln": {"umln": False},
    "no_txt_cond": {"use_txt_cond": False},
    "all_off": _OFF4,
    "prodiff_no_emo_style": dict(PRODIFF_OVERRIDES, emo=False, style=False),
    "conv_no_style": dict(CONVF0_OVERRIDES, style=False),
}
SWITCH_DUR_CONFIG = "all_off"  # the configuration that also stores a forward with predicted durations


def case_switches(name, T=4, frames=32, phones=4, ref_frames=32, seed=151, utt_idx=107):
    """The reference's StyleSinger under each model-switch configuration (stylesinger.py:53-64,92-117,119-187,313-331):
    per configuration the state dict's key list (the synthetic checkpoint loads with strict=True) and a B = 1 full forward
    at T = f0_T = 4 with injected noise, mel2ph given.  emo_embed is passed as None without emo, as forward_model does
    (inference/StyleSinger.py:44-47).  Stored per configuration c as c/<output>; c/coarse_mel (DiffSinger configurations)
    comes from a second run below diff_start.  SWITCH_DUR_CONFIG also stores the forward with predicted durations
    (c/dur_*)."""
    import ref_import
    u = synth.make_utterance(frames / 187.5, utt_idx=utt_idx, ref_frames=ref_frames, frames=frames, phones=phones)
    d, cfg_meta = {}, {}
    for c, ov in SWITCH_CONFIGS.items():
        hp = ref_import.install(T=T, f0_T=T, overrides=ov)
        import modules.diff.shallow_diffusion_tts as sdt
        import modules.diff.gaussian_multinomial_diffusion as gmd
        import modules.diff.prodiff as pdm
        sdt.tqdm = gmd.tqdm = pdm.tqdm = lambda it, **k: it
        from modules.StyleSinger.stylesinger import StyleSinger
        model = StyleSinger(_Dict()).eval()
        model.load_state_dict(synth.acoustic_state_dict(dict(hp), seed=0), strict=True)

        def run(seed_, mel2ph=True, global_steps=320000):
            ns = NoiseSource(seed_)
            b = batchify(u)
            cap, hooks = {}, []
            if hp["style"]:
                hooks.append(model.style_extractor.rqvae.register_forward_hook(
                    lambda m, i, o: cap.__setitem__("rq_in", i[0].detach().clone())))
            with torch.no_grad(), patched_rng(ns):
                out = model(b["txt_tokens"], mel2ph=u["mel2ph"][None] if mel2ph else None, spk_embed=b["spk_embed"],
                            emo_embed=b["emo_embed"] if hp["emo"] else None, ref_mels=b["ref_mels"].clone(),
                            ref_f0=b["ref_f0"].clone(), global_steps=global_steps, infer=True, note=b["note"],
                            note_dur=b["note_dur"], note_type=b["note_type"])
                if hp["style"]:
                    out["rq_codes"] = model.style_extractor.rqvae.quantize(cap["rq_in"])[1]
            for h in hooks:
                h.remove()
            return out, ns.log

        out, log = run(seed)
        keys = ["mel_out", "f0_denorm", "pitch_pred", "decoder_inp", "spk_embed"]
        keys += ["emo_embed"] if hp["emo"] else []
        keys += ["style"] if hp["style"] else []
        for k in keys:
            d[f"{c}/{k}"] = np32(out[k][0])
        if hp["style"]:
            d[f"{c}/rq_codes"] = out["rq_codes"][0].numpy().astype(np.int64)
        if hp["decoder"] == "diffsinger":
            coarse, _ = run(seed, global_steps=50000)  # forcing < global_steps < diff_start: the coarse mel only
            d[f"{c}/coarse_mel"] = np32(coarse["mel_out"][0])
        cfg_meta[c] = {"overrides": ov, "noise_log": log,
                       "state_dict": [[k, list(v.shape)] for k, v in model.state_dict().items()]}
        if c == SWITCH_DUR_CONFIG:
            o2, log2 = run(seed + 1, mel2ph=False)
            d.update({f"{c}/dur_mel2ph": o2["mel2ph"][0].numpy().astype(np.int64), f"{c}/dur_logdur": np32(o2["dur"][0]),
                      f"{c}/dur_mel_out": np32(o2["mel_out"][0]), f"{c}/dur_f0_denorm": np32(o2["f0_denorm"][0])})
            cfg_meta[c]["dur_noise_log"] = log2
    d["meta"] = json.dumps({"T": T, "frames": frames, "phones": phones, "ref_frames": ref_frames, "seed": seed,
                            "utt_idx": utt_idx, "dur_config": SWITCH_DUR_CONFIG, "configs": cfg_meta})
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, len(d), "arrays")


# decoder 'fft' and use_spk_id (stylesinger.py:185-186, fs2.py:37-43): name -> hparams overrides
FFT_SPKID_CONFIGS = {
    "fft_gmdiff": {"decoder": "fft"},
    "fft_conv": dict(CONVF0_OVERRIDES, decoder="fft"),
    "spkid_diffsinger": {"use_spk_id": True},
    "spkid_fft": {"decoder": "fft", "use_spk_id": True},
    "fft_no_emo_style": {"decoder": "fft", "emo": False, "style": False},
}
FFT_SPKID_DUR_CONFIG = "spkid_fft"  # the configuration that also stores a forward with predicted durations
FFT_SPKID_SPEAKER = 37  # the speaker id the use_spk_id configurations look up (num_spk = 150: rows 0 .. 150)


def case_fft_spkid(name, T=4, frames=32, phones=4, ref_frames=32, seed=161, utt_idx=108):
    """The reference's StyleSinger with the FastSpeech 2 mel decoder (decoder 'fft') and with speaker ids (use_spk_id), in
    the layout of ref_switches.npz: per configuration the state dict's key list (strict=True load) and a B = 1 full
    forward at T = f0_T = 4 with injected noise, mel2ph given; c/coarse_mel for the DiffSinger configuration (a run below
    diff_start).  A use_spk_id model gets spk_embed = LongTensor([FFT_SPKID_SPEAKER]), as the reference's forward receives
    it; the others the utterance's speaker vector.  FFT_SPKID_DUR_CONFIG also stores the forward with predicted durations."""
    import ref_import
    u = synth.make_utterance(frames / 187.5, utt_idx=utt_idx, ref_frames=ref_frames, frames=frames, phones=phones)
    d, cfg_meta = {}, {}
    for c, ov in FFT_SPKID_CONFIGS.items():
        hp = ref_import.install(T=T, f0_T=T, overrides=ov)
        import modules.diff.shallow_diffusion_tts as sdt
        import modules.diff.gaussian_multinomial_diffusion as gmd
        sdt.tqdm = gmd.tqdm = lambda it, **k: it
        from modules.StyleSinger.stylesinger import StyleSinger
        model = StyleSinger(_Dict()).eval()
        # (extended_models: the opt-in stylesinger_b200 needs for these options; the reference has no such key)
        model.load_state_dict(synth.acoustic_state_dict(dict(hp, extended_models=True), seed=0), strict=True)
        spk = torch.tensor([FFT_SPKID_SPEAKER]) if hp["use_spk_id"] else u["spk_embed"][None]

        def run(seed_, mel2ph=True, global_steps=320000):
            ns = NoiseSource(seed_)
            b = batchify(u)
            cap, hooks = {}, []
            if hp["style"]:
                hooks.append(model.style_extractor.rqvae.register_forward_hook(
                    lambda m, i, o: cap.__setitem__("rq_in", i[0].detach().clone())))
            with torch.no_grad(), patched_rng(ns):
                out = model(b["txt_tokens"], mel2ph=u["mel2ph"][None] if mel2ph else None, spk_embed=spk,
                            emo_embed=b["emo_embed"] if hp["emo"] else None, ref_mels=b["ref_mels"].clone(),
                            ref_f0=b["ref_f0"].clone(), global_steps=global_steps, infer=True, note=b["note"],
                            note_dur=b["note_dur"], note_type=b["note_type"])
                if hp["style"]:
                    out["rq_codes"] = model.style_extractor.rqvae.quantize(cap["rq_in"])[1]
            for h in hooks:
                h.remove()
            return out, ns.log

        out, log = run(seed)
        keys = ["mel_out", "f0_denorm", "pitch_pred", "decoder_inp", "spk_embed"]
        keys += ["emo_embed"] if hp["emo"] else []
        keys += ["style"] if hp["style"] else []
        for k in keys:
            d[f"{c}/{k}"] = np32(out[k][0])
        if hp["style"]:
            d[f"{c}/rq_codes"] = out["rq_codes"][0].numpy().astype(np.int64)
        if hp["decoder"] == "diffsinger":
            coarse, _ = run(seed, global_steps=50000)  # forcing < global_steps < diff_start: the coarse mel only
            d[f"{c}/coarse_mel"] = np32(coarse["mel_out"][0])
        cfg_meta[c] = {"overrides": ov, "noise_log": log,
                       "state_dict": [[k, list(v.shape)] for k, v in model.state_dict().items()]}
        if c == FFT_SPKID_DUR_CONFIG:
            o2, log2 = run(seed + 1, mel2ph=False)
            d.update({f"{c}/dur_mel2ph": o2["mel2ph"][0].numpy().astype(np.int64), f"{c}/dur_logdur": np32(o2["dur"][0]),
                      f"{c}/dur_mel_out": np32(o2["mel_out"][0]), f"{c}/dur_f0_denorm": np32(o2["f0_denorm"][0])})
            cfg_meta[c]["dur_noise_log"] = log2
    d["meta"] = json.dumps({"T": T, "frames": frames, "phones": phones, "ref_frames": ref_frames, "seed": seed,
                            "utt_idx": utt_idx, "dur_config": FFT_SPKID_DUR_CONFIG, "spk_id": FFT_SPKID_SPEAKER,
                            "configs": cfg_meta})
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, len(d), "arrays")


def case_registry(name, T=4, seed=131):
    """The reference's per-registry modules that the C ABI replaces one by one (FS_ENCODERS['fft'], FS_DECODERS['fft'],
    StyleSinger.get_style): FastspeechEncoder.forward and FastspeechDecoder.forward on padded B = 3 batches and on each
    utterance alone, and get_style at B = 1 (a padded get_style batch is not B = 1-equal in the reference: its padding rows
    are quantised and attended to)."""
    model, hp, sd = build_reference_model(T)
    d_in = registry_inputs(seed)
    with torch.no_grad():
        enc = model.encoder(d_in["enc_tokens"])
        dec = model.decoder(d_in["dec_x"])
        d = {"enc_out": np32(enc), "dec_out": np32(dec)}
        # each utterance alone (B = 1) on its rows up to the last non-padding one
        tok, x = d_in["enc_tokens"], d_in["dec_x"]
        for b in range(3):
            n = int((tok[b] != 0).nonzero()[-1]) + 1
            d[f"enc_b1_{b}"] = np32(model.encoder(tok[b:b + 1, :n])[0])
            n = int((x[b].abs().sum(-1) > 0).nonzero()[-1]) + 1
            d[f"dec_b1_{b}"] = np32(model.decoder(x[b:b + 1, :n])[0])
        for i in range(2):
            ret = {"ref_f0": d_in[f"style_f0_{i}"].clone()}
            d[f"style_{i}"] = np32(model.get_style(d_in[f"style_dec_{i}"], d_in[f"style_ref_{i}"].clone(), ret, infer=True,
                                                   global_steps=320000)[0])
    # the tests regenerate the inputs from the seed; their first values are kept to check that
    d["in_enc_tokens"] = d_in["enc_tokens"].numpy().astype(np.int64)
    d["in_dec_x_head"] = np32(d_in["dec_x"][:, :2, :4])
    d["meta"] = json.dumps({"T": T, "seed": seed})
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, {k: (v.shape if hasattr(v, "shape") else "meta") for k, v in d.items()})


def case_schedules(name, Ts=(4, 25, 50, 100, 200, 500)):
    """Registered schedule buffers of the reference's DiffusionDecoder / GaussianMultinomialDiffusion at several T
    (shallow_diffusion_tts.py:86-119, gaussian_multinomial_diffusion.py:237-283): pins the oracle's and the product's
    independently written schedule code, incl. the T values of BASELINE.json configs[4]."""
    gk = ["betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod",
          "log_one_minus_alphas_cumprod", "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_variance",
          "posterior_log_variance_clipped", "posterior_mean_coef1", "posterior_mean_coef2"]
    mk = ["log_alpha", "log_1_min_alpha", "log_cumprod_alpha", "log_1_min_cumprod_alpha"]
    d = {"Ts": np.asarray(Ts, np.int64)}
    for T in Ts:
        model, hp, _ = build_reference_model(T)
        for k in gk:
            d[f"mel_T{T}_{k}"] = np32(getattr(model.postdiff, k))
            d[f"f0_T{T}_{k}"] = np32(getattr(model.f0_gen, k))
        for k in mk:
            d[f"f0_T{T}_{k}"] = np32(getattr(model.f0_gen, k))
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, len(d), "arrays")


def case_emotion_encoder(name, partials=5, seed=71):
    """f3: the reference's own EmotionEncoder (data_gen/tts/emotion/model.py:10-77, the network behind `emo_embed`,
    inference/StyleSinger.py:106) with seeded random weights on seeded random 160-frame x 40-channel partials:
    `inference` (= hidden[-1], what data_gen/tts/emotion/inference.py:54 uses), `forward` (relu(linear) L2-normalised) and
    the utterance embedding of embed_utterance (inference.py:150-151: mean of the partial embeddings, L2-normalised)."""
    import ref_import
    ref_import.install(T=4)  # reference on sys.path + import shims (hparams unused by the encoder)
    from data_gen.tts.emotion.model import EmotionEncoder
    from oracle.frontend_oracle import emotion_encoder_weights
    cpu = torch.device("cpu")
    model = EmotionEncoder(cpu, cpu).eval()
    # weights: numpy legacy RandomState stream (stable across versions), loaded the stock way; the fixture then only holds
    # inputs and outputs and the tests regenerate the same weights from the seed
    sd = emotion_encoder_weights(seed)
    missing = model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=False)
    assert not [k for k in missing.missing_keys if k.startswith(("lstm.", "linear."))], missing
    g = torch.Generator().manual_seed(seed + 1)
    frames = (torch.randn(partials, 160, 40, generator=g).abs() * 0.3).float()
    with torch.no_grad():
        hidden = model.inference(frames)
        embeds = model.forward(frames)
        frames2 = (torch.randn(3, 97, 40, generator=g).abs() * 2.0).float()  # another length, louder input
        hidden2 = model.inference(frames2)
    raw = hidden.numpy().mean(axis=0)
    d = {"frames2": np32(frames2), "hidden2": np32(hidden2), "seed": np.int64(seed), "frames": np32(frames), "hidden": np32(hidden), "embeds": np32(embeds),
         "utt_embed": (raw / np.linalg.norm(raw, 2)).astype(np.float32)}
    # partial-utterance slicing (inference.py:58-107) for a spread of lengths incl. the short / coverage-edge cases
    from data_gen.tts.emotion.inference import compute_partial_slices
    ns = [1, 159, 160, 8000, 19199, 19200, 25599, 25600, 31999, 32000, 38400, 44799, 44800, 48000, 160000, 163840, 479999]
    rows = []
    for n in ns:
        wav_sl, mel_sl = compute_partial_slices(n)
        for w, m in zip(wav_sl, mel_sl):
            rows.append([n, w.start, w.stop, m.start, m.stop])
    d["slices"] = np.asarray(rows, np.int64)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **d)
    print("wrote", name, len(d), "arrays")


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    which = sys.argv[1:] or ["small", "t25", "t100", "padded", "plms", "prodiff", "convf0", "sched", "voc",
                             "vocoder_edges", "emo", "registry", "kstep", "vocoder_layouts", "switches", "fft_spkid"]
    if "small" in which:
        case_model("ref_small_T4", T=4, frames=96, phones=12, ref_frames=64, seed=11, utt_idx=100)
    if "t25" in which:
        case_model("ref_f64_T25", T=25, frames=64, phones=8, ref_frames=48, seed=21, utt_idx=101, with_dur_case=False)
    if "t100" in which:  # the bench's step count (T=100 mel + 2 x 100 F0 steps) on a tiny utterance
        case_model("ref_f32_T100", T=100, frames=32, phones=4, ref_frames=32, seed=41, utt_idx=102, with_dur_case=False)
    if "padded" in which:
        case_padded("ref_padded_T4")
    if "plms" in which:
        case_plms("ref_plms_T100_i10")
    if "prodiff" in which:
        case_prodiff("ref_prodiff_T8")
    if "convf0" in which:
        case_convf0("ref_convf0")
    if "sched" in which:
        case_schedules("ref_schedules")
    if "voc" in which:
        case_vocoder("ref_vocoder_f24", frames=24, seed=31)
    if "vocoder_edges" in which:
        case_vocoder_edges("ref_vocoder_edges")
    if "vocoder_layouts" in which:
        case_vocoder_layouts("ref_vocoder_layouts")
    if "emo" in which:
        case_emotion_encoder("ref_emotion_encoder")
    if "registry" in which:
        case_registry("ref_registry")
    if "kstep" in which:
        case_kstep("ref_kstep")
    if "switches" in which:
        case_switches("ref_switches")
    if "fft_spkid" in which:
        case_fft_spkid("ref_fft_spkid")
