"""Reference-named module facades over libstylesinger_b200.so (inference only).

``StyleSinger`` mirrors ``modules/StyleSinger/stylesinger.py:119-187`` (``forward`` keyword arguments, padded
[B, L, ...] tensors in, the ``ret`` dict the reference's callers read out: inference/StyleSinger.py:54-55,
tasks/StyleSinger/stylesinger.py:122-123,190-195).  ``HifiGAN`` mirrors the registered vocoder class
(tasks/tts/vocoder_infer/hifigan_nsf.py:46-75: ``spec2wav(mel np[T,80], f0=np[T]) -> np[T*hop]``).

The three mel decoders of ``hparams['decoder']`` are implemented: 'diffsinger' (the default), 'prodiff', the ProDiff
teacher (stylesinger.py:111-117,176-177), whose sampler always runs, whatever ``global_steps`` is, and 'fft', the
FastSpeech 2 decoder alone (:185-186), whose mel is the output at any ``global_steps``.  Both F0 generators of
``hparams['f0_gen']`` are implemented: 'gmdiff' (the default) and 'conv' (stylesinger.py:73-82; ``PitchPredictor``).
With ``hparams['use_spk_id']`` the ``spk_embed`` argument is a LongTensor [B] of speaker ids, as the reference's forward
receives it (fs2.py:37-38).  'fft' and use_spk_id need ``hparams['extended_models'] = True``.  Only what the ph -> mel -> wav inference path uses is implemented; everything else raises
instead of silently doing something different (training mode, teacher-forced f0/uv, the `forcing` aligner branch of
early training steps).
"""
from typing import Dict, List, Optional

import numpy as np
import torch

from .engine import AcousticModel, PackedBatch, Vocoder, pack_batch, utt_seeds
from .hparams import resolve


def padded_to_utterances(txt_tokens, note, note_dur, note_type, spk_embed, emo_embed, ref_mels, ref_f0,
                         mel2ph=None, spk_id=False) -> List[Dict[str, torch.Tensor]]:
    """Split the reference's zero-padded batch tensors into per-utterance true-length CPU tensors.

    Padding conventions of the reference collater (tasks/StyleSinger/dataset.py): token id 0 pads ``txt_tokens``
    (and the note tensors alongside), all-zero frames pad ``ref_mels`` (the reference derives its own mask from
    ``ref_mels[:, :, 0] != 0``, lse.py:104, and so does the kernel), 0 pads ``mel2ph``.
    ``emo_embed`` None (a model without emo) or ``ref_mels`` None (without style) leaves those fields out.
    ``spk_id``: ``spk_embed`` holds one integer speaker id per batch row (use_spk_id), stored as ``u["spk_id"]``.
    """
    txt_tokens = torch.as_tensor(txt_tokens).cpu()
    B = txt_tokens.shape[0]
    if ref_mels is not None:
        ref_mels = torch.as_tensor(ref_mels).float().cpu()
        ref_f0 = torch.as_tensor(ref_f0).float().cpu()
        if ref_f0.dim() == 1:  # inference/StyleSinger.py passes [R] at B=1
            ref_f0 = ref_f0[None]
    utts = []
    for b in range(B):
        nz = (txt_tokens[b] != 0).nonzero()
        P = int(nz[-1]) + 1 if len(nz) else 0
        if P == 0:
            raise ValueError(f"utterance {b}: empty phone sequence")
        u = {"txt_tokens": txt_tokens[b, :P].long(), "note": torch.as_tensor(note)[b, :P].long().cpu(),
             "note_dur": torch.as_tensor(note_dur)[b, :P].float().cpu(),
             "note_type": torch.as_tensor(note_type)[b, :P].long().cpu()}
        if spk_id:
            u["spk_id"] = int(torch.as_tensor(spk_embed).reshape(B)[b])
        else:
            u["spk_embed"] = torch.as_tensor(spk_embed)[b].float().reshape(-1).cpu()
        if emo_embed is not None:
            u["emo_embed"] = torch.as_tensor(emo_embed)[b].float().reshape(-1).cpu()
        if ref_mels is not None:
            rnz = (ref_mels[b].abs().sum(-1) > 0).nonzero()
            R = int(rnz[-1]) + 1 if len(rnz) else 0
            if R == 0:
                raise ValueError(f"utterance {b}: empty reference mel")
            u["ref_mels"], u["ref_f0"] = ref_mels[b, :R], ref_f0[b, :R]
        if mel2ph is not None:
            m2p = torch.as_tensor(mel2ph)[b].long().cpu()
            fnz = (m2p != 0).nonzero()
            F = int(fnz[-1]) + 1 if len(fnz) else 0
            if F == 0:
                raise ValueError(f"utterance {b}: empty mel2ph")
            u["mel2ph"] = m2p[:F]
        utts.append(u)
    return utts


def packed_to_padded(x: torch.Tensor, offsets, pad_value=0) -> torch.Tensor:
    """Tight [sum_L, ...] rows + host offsets [B+1] -> zero-padded [B, max_L, ...] (the reference's layout)."""
    B = len(offsets) - 1
    lens = [int(offsets[i + 1] - offsets[i]) for i in range(B)]
    out = x.new_full((B, max(lens) if lens else 0) + tuple(x.shape[1:]), pad_value)
    for i in range(B):
        out[i, :lens[i]] = x[int(offsets[i]):int(offsets[i + 1])]
    return out


class StyleSinger:
    """Inference facade with the reference module's call signature (``model(txt_tokens, ..., infer=True)``)."""

    RET_KEYS = ("mel_out", "f0_denorm", "mel2ph", "decoder_inp", "style", "pitch_pred", "spk_embed", "emo_embed",
                "x_mask", "dur")

    def __init__(self, state_dict=None, hparams=None, device=None, engine: Optional[AcousticModel] = None):
        self.hparams = resolve(hparams)
        self.engine = engine if engine is not None else AcousticModel(state_dict, self.hparams, device)
        self.training = False

    def eval(self):
        return self

    def to(self, *a, **k):  # the reference driver calls model.to(device); the engine already lives on its GPU
        return self

    def __call__(self, *args, **kwargs):
        return self.forward(*args, **kwargs)

    def get_style(self, encoder_out, ref_mels, ret, infer=False, global_steps=0):
        """modules/StyleSinger/stylesinger.py:189-214 with padded tensors (ret['ref_f0'] as there)."""
        dev = self.engine.device
        fl = _true_lengths(encoder_out)
        rl = _true_lengths(ref_mels)
        fo = np.concatenate([[0], np.cumsum(fl)]).astype(np.int32)
        ro = np.concatenate([[0], np.cumsum(rl)]).astype(np.int32)
        rf0 = ret["ref_f0"]
        rf0 = rf0[None] if rf0.dim() == 1 else rf0
        dec = torch.cat([encoder_out[i, :n] for i, n in enumerate(fl)]).to(dev, torch.float32).contiguous()
        rm = torch.cat([ref_mels[i, :n] for i, n in enumerate(rl)]).to(dev, torch.float32).contiguous()
        rf = torch.cat([rf0[i, :n] for i, n in enumerate(rl)]).to(dev, torch.float32).contiguous()
        style, _ = self.engine.get_style(dec, fo, rm, rf, ro)
        ret["rq_loss"], ret["gloss"] = 0.0, 0.0
        out = packed_to_padded(style, fo)
        if out.shape[1] < encoder_out.shape[1]:
            out = torch.cat([out, out.new_zeros(out.shape[0], encoder_out.shape[1] - out.shape[1], out.shape[2])], 1)
        return out

    def forward(self, txt_tokens, mel2ph=None, spk_embed=None, emo_embed=None, ref_mels=None, ref_f0=None,
                f0=None, uv=None, skip_decoder=False, global_steps=0, infer=False, note=None, note_dur=None,
                note_type=None, seed=0, noise=None, seeds=None, **kwargs):
        """seeds: one seed per batch row instead of `seed` (AcousticModel.forward): row b then gets the outputs of the
        B = 1 call with seed=seeds[b]."""
        hp = self.hparams
        if seeds is not None:  # checked before anything reaches the device
            seeds = utt_seeds(seeds, txt_tokens.shape[0])
            if noise is not None:
                raise ValueError("seeds: per-utterance seeds key the in-kernel noise; noise must be None")
        if not infer:
            raise NotImplementedError("stylesinger_b200 implements the inference path only (infer=True)")
        if f0 is not None or uv is not None:
            raise NotImplementedError("teacher-forced f0/uv is a training-time input; the inference path predicts pitch")
        if global_steps < hp.get("forcing", 0):
            raise NotImplementedError("global_steps < hparams['forcing'] selects the forced-alignment branch of "
                                      "ProsodyAligner (training warm-up); pass the checkpoint's step count")
        if hp["emo"] and hp["style"]:
            if spk_embed is None or emo_embed is None or ref_mels is None or ref_f0 is None or note is None:
                raise ValueError("spk_embed, emo_embed, ref_mels, ref_f0 and note/note_dur/note_type are required")
        else:  # the model switches decide what the model reads (stylesinger.py:131-137,149-151)
            need = {"spk_embed": spk_embed, "note": note}
            if hp["emo"]:
                need["emo_embed"] = emo_embed
            if hp["style"]:
                need.update(ref_mels=ref_mels, ref_f0=ref_f0)
            missing = [k for k, v in need.items() if v is None]
            if missing:
                raise ValueError(f"{', '.join(missing)} required by this model (hparams emo={hp['emo']}, "
                                 f"style={hp['style']})")
        # a switched-off module's input is not read, whatever the caller passes (the reference ignores it too)
        utts = padded_to_utterances(txt_tokens, note, note_dur, note_type, spk_embed, emo_embed if hp["emo"] else None,
                                    ref_mels if hp["style"] else None, ref_f0 if hp["style"] else None, mel2ph,
                                    spk_id=hp["use_spk_id"])
        pb: PackedBatch = pack_batch(utts, use_mel2ph=mel2ph is not None, emo=hp["emo"], style=hp["style"],
                                     spk_id=hp["use_spk_id"]).to(self.engine.device)
        ret = {}
        dur = None
        if pb.frame_offsets is None:  # FastSpeech2.add_dur at inference (fs2.py:151-174): predicted durations
            dur, _ = self.engine.predict_durations(pb)
            d = dur.cpu().numpy()
            po = pb.ph_offsets
            lens = [int(d[po[i]:po[i + 1]].sum()) for i in range(pb.B)]
            pb.frame_offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
            ret["dur"] = packed_to_padded(dur, po)
        # the reference runs the shallow-diffusion refinement only once training passed diff_start (stylesinger.py:181);
        # the ProDiff branch has no such gate and no coarse mel (:176-177), and the FFT decoder's mel is always the output
        # (:185-186)
        ungated = hp["decoder"] in ("prodiff", "fft")
        run_diff = (not skip_decoder) and (ungated or global_steps > hp.get("diff_start", 0))
        want = ["f0_denorm", "mel2ph", "decoder_inp", "pitch_pred", "spk_proj"]
        want += ["emo_proj"] if hp["emo"] else []
        want += ["style"] if hp["style"] else []
        if not skip_decoder:
            want.append("mel_out" if run_diff else "coarse_mel")
        if callable(noise):  # parity hooks: the injected draws depend on the (possibly predicted) frame count
            noise = noise(pb.frame_offsets)
        keyed = {} if seeds is None else {"seeds": seeds}
        out = self.engine.forward(pb, noise=noise, seed=seed, skip_mel_diffusion=not run_diff, dur=dur, want=tuple(want),
                                  **keyed)
        fo = pb.frame_offsets
        m2p = packed_to_padded(out["mel2ph"].long(), fo)
        ret["mel2ph"] = m2p
        ret["x_mask"] = (m2p > 0).float()[:, :, None]
        ret["f0_denorm"] = packed_to_padded(out["f0_denorm"], fo)
        ret["decoder_inp"] = packed_to_padded(out["decoder_inp"], fo)
        if hp["style"]:  # the reference sets ret['style'] only then (stylesinger.py:149-151)
            ret["style"] = packed_to_padded(out["style"], fo)
        ret["pitch_pred"] = packed_to_padded(out["pitch_pred"], fo)
        ret["spk_embed"] = out["spk_proj"][:, None, :]
        if hp["emo"]:  # the reference sets ret['emo_embed'] only then (stylesinger.py:131-132)
            ret["emo_embed"] = out["emo_proj"][:, None, :]
        if not skip_decoder:
            ret["mel_out"] = packed_to_padded(out["mel_out" if run_diff else "coarse_mel"], fo)
        # training-only entries the callers index unconditionally
        for k in ("gdiff1", "gdiff2", "mdiff1", "mdiff2", "diff", "rq_loss", "gloss"):
            ret[k] = 0.0
        return ret


def _lengths_from_mask(nz: torch.Tensor):
    """Per batch element of a [B, L] non-padding mask, the index after its last True (at least 1).  Padding only ever
    trails, so this is the true length; an interior padding row stays inside it, where the library masks it exactly as
    the reference does (a count of the True entries would drop the last real row instead)."""
    L = nz.shape[1]
    idx = torch.arange(1, L + 1, device=nz.device)[None, :] * nz
    return [max(int(v), 1) for v in idx.max(dim=1).values.tolist()]


def _true_lengths(x: torch.Tensor):
    """Per batch element, the index after the last row that is not all zero (the reference's padding rows are zero)."""
    return _lengths_from_mask(x.abs().sum(-1) > 0)


class _Registered(torch.nn.Module):
    """Common shell of the per-registry drop-ins: parameter-free nn.Modules (the reference assigns them where it holds
    child modules, and calls .eval() / .to(device) on the tree); the weights live in the engine's packed model."""

    def __init__(self, engine: AcousticModel):
        super().__init__()
        object.__setattr__(self, "engine", engine)


class FastspeechEncoder(_Registered):
    """FS_ENCODERS['fft'] drop-in (modules/fastspeech/fs2.py:9-13): ``forward(txt_tokens [B,T]) -> [B,T,256]``."""

    def forward(self, txt_tokens):
        dev = self.engine.device
        lens = _lengths_from_mask(txt_tokens != 0)  # pad id 0 (dictionary.pad())
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        tight = torch.cat([txt_tokens[i, :n] for i, n in enumerate(lens)]).to(dev, torch.int32).contiguous()
        out = self.engine.fft_encoder(tight, offs)
        pad = packed_to_padded(out, offs)
        if pad.shape[1] < txt_tokens.shape[1]:
            pad = torch.cat([pad, pad.new_zeros(pad.shape[0], txt_tokens.shape[1] - pad.shape[1], pad.shape[2])], 1)
        return pad


class FastspeechDecoder(_Registered):
    """FS_DECODERS['fft'] drop-in (modules/fastspeech/fs2.py:15-18): ``forward(x [B,T,256]) -> [B,T,256]``."""

    def forward(self, x, padding_mask=None, attn_mask=None, return_hiddens=False):
        if padding_mask is not None or attn_mask is not None or return_hiddens:
            raise NotImplementedError("FastspeechDecoder drop-in: only forward(x) (the call the StyleSinger path makes)")
        dev = self.engine.device
        lens = _true_lengths(x)
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        tight = torch.cat([x[i, :n] for i, n in enumerate(lens)]).to(dev, torch.float32).contiguous()
        out = packed_to_padded(self.engine.fft_decoder(tight, offs), offs)
        if out.shape[1] < x.shape[1]:
            out = torch.cat([out, out.new_zeros(out.shape[0], x.shape[1] - out.shape[1], out.shape[2])], 1)
        return out


class DiffNet(_Registered):
    """DIFF_DECODERS['wavenet'] drop-in (modules/StyleSinger/stylesinger.py:38-40), called by the reference's sampler as
    ``denoise_fn(spec [B,1,M,F], diffusion_step [B], cond [B,H,F]) -> [B,1,M,F]`` (shallow_diffusion_tts.py:146)."""

    def forward(self, spec, diffusion_step, cond):
        B, _, M, Fr = spec.shape
        t = int(diffusion_step.reshape(-1)[0])
        offs = (np.arange(B + 1) * Fr).astype(np.int32)
        x = spec[:, 0].transpose(1, 2).reshape(B * Fr, M).to(self.engine.device, torch.float32).contiguous()
        c = cond.transpose(1, 2).reshape(B * Fr, cond.shape[1]).to(self.engine.device, torch.float32).contiguous()
        out = self.engine.denoiser_eval(0, x, None, t, c, offs)
        return out.reshape(B, Fr, M).transpose(1, 2)[:, None].contiguous()


class DDiffNet(_Registered):
    """Drop-in for the two F0/UV denoisers (modules/diff/net.py:215-266), called from
    GaussianMultinomialDiffusion.sample (gaussian_multinomial_diffusion.py:930-935) as
    ``denoise_fn(f0 [B,1,F], uv [B,F] long, diffusion_step [B], cond [B,H,F], nonpadding [B,F]) -> [B,3,F]``.
    which: 1 = gm_diffnet (domain-agnostic), 2 = gm_diffnet_inpainte (domain-specific)."""

    def __init__(self, engine: AcousticModel, which: int):
        super().__init__(engine)
        self.which = which

    def forward(self, f0, uv, diffusion_step, cond, nonpadding=None):
        B, _, Fr = f0.shape
        t = int(diffusion_step.reshape(-1)[0])
        offs = (np.arange(B + 1) * Fr).astype(np.int32)
        dev = self.engine.device
        x = f0.reshape(B * Fr).to(dev, torch.float32).contiguous()
        u = uv.reshape(B * Fr).to(dev, torch.int32).contiguous()
        c = cond.transpose(1, 2).reshape(B * Fr, cond.shape[1]).to(dev, torch.float32).contiguous()
        out = self.engine.denoiser_eval(self.which, x, u, t, c, offs)  # [B*F, 3]
        out = out.reshape(B, Fr, 3).transpose(1, 2).contiguous()
        return out if nonpadding is None else out * nonpadding[:, None, :].to(out.device)


class PitchPredictor(_Registered):
    """Drop-in for the two FastSpeech-2 PitchPredictors of an f0_gen 'conv' model (stylesinger.py:73-82,223-225;
    tts_modules.py:191-234): ``forward(xs [B,T,256]) -> [B,T,2]`` (log2-Hz f0, uv logit).  which: 0 = pitch_predictor
    (domain agnostic), 1 = pitch_inpainter_predictor (domain specific).  The reference applies no mask inside the
    predictor, so every batch element runs over the full padded length T, exactly as the reference computes it."""

    def __init__(self, engine: AcousticModel, which: int):
        super().__init__(engine)
        self.which = which

    def forward(self, xs):
        B, T, H = xs.shape
        offs = (np.arange(B + 1) * T).astype(np.int32)
        x = xs.reshape(B * T, H).to(self.engine.device, torch.float32).contiguous()
        return self.engine.pitch_predictor(self.which, x, offs).reshape(B, T, 2)


class HifiGAN:
    """``spec2wav(mel, f0=...)`` with numpy in / numpy out (tasks/tts/vocoder_infer/hifigan_nsf.py:62-75).  ``denoise_c`` is
    hparams['vocoder_denoise_c']: > 0 runs the reference's output denoiser (:14-22,73-74) on the waveform.
    ``tc_precision`` is hparams['tc_precision'] ('split' or 'fp16') of the vocoder this facade creates; a given ``engine``
    keeps its own (Vocoder.set_precision)."""

    def __init__(self, state_dict=None, config=None, device=None, use_nsf=True, engine: Optional[Vocoder] = None,
                 denoise_c=0.0, tc_precision="split"):
        self.v = engine if engine is not None else Vocoder(state_dict, config, device, tc_precision=tc_precision)
        self.use_nsf = use_nsf
        self.denoise_c = float(denoise_c)

    def spec2wav(self, mel, **kwargs):
        f0 = kwargs.get("f0")
        dev = self.v.device
        m = torch.as_tensor(np.ascontiguousarray(mel), dtype=torch.float32).to(dev)
        f = None
        if f0 is not None and self.use_nsf:
            f = torch.as_tensor(np.ascontiguousarray(f0), dtype=torch.float32).to(dev)
        offs = np.array([0, m.shape[0]], np.int32)
        wav = self.v.generate(m, f, offs, seed=int(kwargs.get("seed", 0)), denoise_c=self.denoise_c)
        return wav.cpu().numpy()
