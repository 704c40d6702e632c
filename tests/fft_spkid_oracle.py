"""FastSpeech 2 mel decoder and speaker-id restatement (test infrastructure, oracle side): StyleSinger.forward(infer=True)
with hparams['decoder'] == 'fft' (reference modules/StyleSinger/stylesinger.py:185-186; run_decoder,
modules/fastspeech/fs2.py:233-237) and with hparams['use_spk_id'] (spk_embed_proj = Embedding(num_spk + 1, 256) looked up
by an integer id, fs2.py:37-43), under every model switch, F0 generator and mel decoder.

Pinned against tests/golden/ref_fft_spkid.npz (dumped from the unmodified reference by tools/make_golden.py fft_spkid) in
tests/test_fft_spkid_cpu.py.  Without either option it is tests/switches_oracle.py's forward; the body is restated here
because that one reads a Linear spk_embed_proj and always ends in a diffusion sampler.  Every piece it calls is the shared
oracle's, the conv-F0 restatement's (tests/f0conv_oracle.py) or the ProDiff restatement's (tests/prodiff_oracle.py).
"""
import torch
import torch.nn.functional as F

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from stylesinger_b200.hparams import resolve
from tests import f0conv_oracle as F0C
from tests import prodiff_oracle as PO

_SD = {}


def switch_hp(cfg):
    """hparams of a fixture configuration, cfg = {"T": ..., "overrides": {...}}, with the opt-in the two options need
    (hparams['extended_models']); without either option it is tests/switches_oracle.py's switch_hp plus that key."""
    return resolve(timesteps=cfg["T"], K_step=cfg["T"], f0_timesteps=cfg["T"], extended_models=True, **cfg["overrides"])


def switch_sd(cfg):
    """The synthetic checkpoint of a configuration (cached)."""
    key = (cfg["T"], tuple(sorted(cfg["overrides"].items())))
    if key not in _SD:
        _SD[key] = synth.acoustic_state_dict(switch_hp(cfg), seed=0)
    return _SD[key]


def speaker(sd, hp, spk):
    """ret['spk_embed'] [B, 1, 256] (stylesinger.py:130): the table rows of the ids spk (LongTensor [B]) with use_spk_id,
    else the Linear over the speaker vectors spk [B, 256]."""
    if hp["use_spk_id"]:
        return F.embedding(spk, sd["spk_embed_proj.weight"])[:, None, :]
    return F.linear(spk, sd["spk_embed_proj.weight"], sd["spk_embed_proj.bias"])[:, None, :]


def stylesinger_forward(sd, hp, txt_tokens, note, note_dur, note_type, spk, emo_embed, ref_mels, ref_f0, noise,
                        mel2ph=None, skip_diffusion=False):
    """StyleSinger.forward(infer=True, global_steps > diff_start) for B = 1.  spk: speaker ids [B] (use_spk_id) or
    speaker vectors [B, 256].  emo_embed is unread without emo, ref_mels / ref_f0 without style.  Draw order: the two F0
    samplers (gmdiff), then the mel sampler (none on an FFT model)."""
    ret = {}
    enc = O.fastspeech_encoder(txt_tokens, sd, hp) + O.note_encoder(note, note_dur, note_type, sd, hp["hidden_size"])
    src_np = (txt_tokens > 0).float()[:, :, None]
    spk = speaker(sd, hp, spk)
    ret["spk_embed"] = spk
    emo = 0.0
    if hp["emo"]:  # :131-132
        emo = F.linear(emo_embed, sd["emo_embed_proj.weight"], sd["emo_embed_proj.bias"])[:, None, :]
        ret["emo_embed"] = emo
    if mel2ph is None:  # dur_inp = (encoder_out + spk [+ emo]) * src_nonpadding (:134-139)
        dur, xs = O.duration_predictor((enc + spk + emo) * src_np, txt_tokens == 0, sd, hp)
        ret["dur"], ret["dur_choice"] = xs, dur
        mel2ph = O.length_regulator(dur, txt_tokens == 0)
    ret["mel2ph"] = mel2ph
    tgt_np = (mel2ph > 0).float()[:, :, None]
    dec = O.expand_states(enc, mel2ph)  # UMLN = identity in eval (umln.py:49-50)
    style = 0.0
    if hp["style"]:  # :149-151
        style, codes = O.get_style(dec, ref_mels, ref_f0, sd, hp)
        ret["style"], ret["rq_codes"] = style, codes
    agn = dec * tgt_np
    spc = (dec + spk + emo + style) * tgt_np  # :157-163
    if hp["f0_gen"] == "conv":
        pit = F0C.inpaint_pitch(agn, spc, mel2ph, sd)
    else:
        midi = O.expand_states(note[:, :, None], mel2ph).transpose(-1, -2)
        pit = O.inpaint_pitch(agn, spc, mel2ph, midi.float(), sd, hp, noise)
    ret.update({"pitch_pred": pit["pitch_pred"], "f0_denorm": pit["f0_denorm"], "pitch": pit["pitch"]})
    dec = (dec + spk + pit["pitch_embed"] + emo + style) * tgt_np  # :167-172
    ret["decoder_inp"] = dec
    if hp["decoder"] == "prodiff":  # :176-177
        if not skip_diffusion:
            ret["mel_out"] = PO.mel_prodiff_sample(dec, sd, hp, noise)
        return ret
    coarse = F.linear(O.fastspeech_decoder(dec, sd, hp), sd["mel_out.weight"], sd["mel_out.bias"]) * tgt_np
    if hp["decoder"] == "fft":  # :185-186: run_decoder's mel is the output
        ret["mel_out"] = coarse
        return ret
    ret["coarse_mel"] = coarse
    Fr = coarse.shape[1]
    g = [coarse] + ([dec] if hp["use_txt_cond"] else []) + [spk.repeat(1, Fr, 1)]  # run_diffsinger (:313-327)
    g += [emo.repeat(1, Fr, 1)] if hp["emo"] else []
    g += [style] if hp["style"] else []
    g = F.linear(torch.cat(g, dim=-1), sd["ln_proj.weight"], sd["ln_proj.bias"])
    ret["diff_cond"] = g
    if not skip_diffusion:
        ret["mel_out"] = O.mel_diffusion_sample(g, coarse, sd, hp, noise)
    return ret
