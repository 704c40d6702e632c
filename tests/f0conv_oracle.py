"""Convolutional F0 generator restatement (test infrastructure, oracle side): what hparams['f0_gen'] == 'conv' selects
(reference modules/StyleSinger/stylesinger.py:73-82,216-247; PitchPredictor, modules/fastspeech/tts_modules.py:191-234).

Pinned against tests/golden/ref_convf0.npz (dumped from the unmodified reference by tools/make_golden.py convf0) in
tests/test_f0conv_cpu.py.  Everything else is the shared oracle (oracle/stylesinger_oracle.py) and the ProDiff
restatement (tests/prodiff_oracle.py), which this module only imports.
"""
import torch
import torch.nn.functional as F

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from stylesinger_b200.hparams import resolve
from tests import prodiff_oracle as PO

PREFIXES = ("pitch_predictor.", "pitch_inpainter_predictor.")  # which = 0 (domain agnostic), 1 (domain specific)
_SD = {}


def conv_hp(meta):
    """hparams of a fixture configuration (meta, or meta['prodiff']): f0_gen 'conv' plus the fixture's overrides."""
    return resolve(timesteps=meta["T"], K_step=meta["T"], **meta["overrides"])


def conv_sd(meta):
    """The synthetic checkpoint the fixture was generated with (cached per configuration)."""
    key = (meta["T"], tuple(sorted(meta["overrides"].items())))
    if key not in _SD:
        _SD[key] = synth.acoustic_state_dict(conv_hp(meta), seed=0)
    return _SD[key]


def predictor_inputs(meta):
    """The seeded inputs of the fixture's predictor-only case: [2, pred_frames, 256] (one per predictor), channel 0
    exactly 0 in the rows meta['pred_zero_rows']."""
    g = torch.Generator().manual_seed(meta["pred_seed"])
    xs = torch.randn(2, 1, meta["pred_frames"], 256, generator=g)
    xs[:, :, meta["pred_zero_rows"], 0] = 0
    return xs[:, 0]


def pitch_predictor(xs, sd, which, dtype=torch.float32):
    """PitchPredictor.forward (tts_modules.py:221-234) in eval mode: xs [B,T,H] -> [B,T,2].  positions come from
    make_positions(xs[..., 0]) (padding_idx 0: a row whose channel 0 is exactly 0 gets the zero row and does not count);
    then 5 x (zero SAME pad, Conv1d, ReLU, channel LayerNorm eps 1e-5); then Linear.  No mask anywhere."""
    p = PREFIXES[which]
    w = {k[len(p):]: v.to(dtype) for k, v in sd.items() if k.startswith(p)}
    H = xs.shape[-1]
    xs = xs.to(dtype)
    pos = O.sinusoid_positions(xs[..., 0].cpu(), H).to(xs.device, dtype)
    x = (xs + w["pos_embed_alpha"] * pos).transpose(1, -1)
    i = 0
    while f"conv.{i}.1.weight" in w:
        k = w[f"conv.{i}.1.weight"].shape[-1]
        x = F.pad(x, ((k - 1) // 2, (k - 1) // 2))
        x = F.relu(F.conv1d(x, w[f"conv.{i}.1.weight"], w[f"conv.{i}.1.bias"]))
        x = O.layer_norm_ch(x, w[f"conv.{i}.3.weight"], w[f"conv.{i}.3.bias"])
        i += 1
    return F.linear(x.transpose(1, -1), w["linear.weight"], w["linear.bias"])


def inpaint_pitch(agn, spc, mel2ph, sd, f0=None, uv=None):
    """StyleSinger.inpaint_pitch, f0_gen 'conv' (stylesinger.py:216-247): no noise, no MIDI band, rests not forced
    unvoiced; f0 = pitch_pred[..., 0] is log2 Hz as is, uv = (averaged logit > 0)."""
    pa = pitch_predictor(agn, sd, 0)
    ps = pitch_predictor(spc, sd, 1)
    pred = ps / 2 + pa / 2
    if f0 is None:
        f0 = pred[:, :, 0]
        uv = pred[:, :, 1] > 0
    f0_denorm = 2 ** f0
    if uv is not None:
        f0_denorm = torch.where(uv > 0, torch.zeros_like(f0_denorm), f0_denorm)
    f0_denorm = torch.where(mel2ph == 0, torch.zeros_like(f0_denorm), f0_denorm)
    pitch = O.f0_to_coarse(f0_denorm)
    emb = F.embedding(pitch, sd["pitch_embed.weight"], padding_idx=0)
    return {"pitch_pred": pred, "f0_denorm": f0_denorm, "pitch": pitch, "pitch_embed": emb,
            "pitch_agnostic": pa, "pitch_specific": ps}


def stylesinger_forward(sd, hp, txt_tokens, note, note_dur, note_type, spk_embed, emo_embed, ref_mels, ref_f0, noise,
                        mel2ph=None, f0=None, uv=None, skip_diffusion=False):
    """StyleSinger.forward(infer=True) with f0_gen 'conv' (stylesinger.py:119-187) for B=1, for either mel decoder
    (hp['decoder']).  The shared oracle's forward hard-wires the gmdiff pitch block, so its body is restated here around
    inpaint_pitch above; every other piece is the shared oracle's.  The only noise drawn is the mel sampler's."""
    ret = {}
    enc = O.fastspeech_encoder(txt_tokens, sd, hp) + O.note_encoder(note, note_dur, note_type, sd, hp["hidden_size"])
    spk = F.linear(spk_embed, sd["spk_embed_proj.weight"], sd["spk_embed_proj.bias"])[:, None, :]
    emo = F.linear(emo_embed, sd["emo_embed_proj.weight"], sd["emo_embed_proj.bias"])[:, None, :]
    if mel2ph is None:
        dur, xs = O.duration_predictor((enc + spk + emo) * (txt_tokens > 0).float()[:, :, None], txt_tokens == 0, sd, hp)
        ret["dur"] = xs
        mel2ph = O.length_regulator(dur, txt_tokens == 0)
    ret["mel2ph"] = mel2ph
    tgt_np = (mel2ph > 0).float()[:, :, None]
    dec = O.expand_states(enc, mel2ph)
    style, _ = O.get_style(dec, ref_mels, ref_f0, sd, hp)
    pit = inpaint_pitch(dec * tgt_np, (dec + spk + emo + style) * tgt_np, mel2ph, sd, f0, uv)
    ret.update({k: pit[k] for k in ("pitch_pred", "f0_denorm", "pitch", "pitch_agnostic", "pitch_specific")})
    dec = (dec + spk + pit["pitch_embed"] + emo + style) * tgt_np
    ret["decoder_inp"] = dec
    if hp["decoder"] == "prodiff":
        if not skip_diffusion:
            ret["mel_out"] = PO.mel_prodiff_sample(dec, sd, hp, noise)
        return ret
    coarse = F.linear(O.fastspeech_decoder(dec, sd, hp), sd["mel_out.weight"], sd["mel_out.bias"]) * tgt_np
    Fr = coarse.shape[1]
    g = torch.cat([coarse, dec, spk.repeat(1, Fr, 1), emo.repeat(1, Fr, 1), style], dim=-1)
    g = F.linear(g, sd["ln_proj.weight"], sd["ln_proj.bias"])
    ret["coarse_mel"] = coarse
    if not skip_diffusion:
        ret["mel_out"] = O.mel_diffusion_sample(g, coarse, sd, hp, noise)
    return ret
