"""Drop-in mirror of the reference's inference driver (reference inference/StyleSinger.py:21-179).

``StyleSingerInfer`` keeps the reference's method names and argument meaning (``forward_model(inp)``
with the dict produced by ``preprocess_input``; ``input_to_batch``) and adds ``infer_batch`` for ragged
batches.  Model + vocoder run in libstylesinger_b200.so; the mel / f0 hand-off between them stays on
the device (the reference round-trips through numpy, inference/StyleSinger.py:54-63).
"""
import ctypes as C
import weakref
from typing import List

import numpy as np
import torch

from ._lib import check, lib
from .engine import AcousticModel, PackedBatch, Vocoder, pack_batch, utt_seeds
from .formats import norm_interp_f0, pad_f0_to_mel
from .hparams import resolve


class StyleSingerInfer:
    def __init__(self, hparams=None, device=None, model_state_dict=None, vocoder_state_dict=None, vocoder_config=None,
                 ph_encoder=None):
        """``model_state_dict`` / ``vocoder_state_dict``: the reference checkpoints' ``state_dict['model']`` and
        ``state_dict['model_gen']`` (utils/commons/ckpt_utils.py:26-67, vocoder_infer/hifigan_nsf.py:24-40)."""
        self.hparams = resolve(hparams)
        self.device = torch.device(device if device is not None else "cuda:0")
        self.ph_encoder = ph_encoder
        if model_state_dict is None or vocoder_state_dict is None:
            raise ValueError("state dicts required (reference checkpoints or stylesinger_b200.synth.*_state_dict)")
        self.model = AcousticModel(model_state_dict, self.hparams, self.device)
        # HifiGAN.spec2wav (tasks/tts/vocoder_infer/hifigan_nsf.py:73-74): denoise the waveform when vocoder_denoise_c > 0
        self.vocoder = Vocoder(vocoder_state_dict, vocoder_config, self.device,
                               denoise_c=self.hparams.get("vocoder_denoise_c", 0.0), denoise_hp=self.hparams,
                               tc_precision=self.hparams["tc_precision"])
        self._cnt = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._pinned = []  # [(pinned tensor, weakref to the numpy array handed out last)]: see _host_out

    def _host_out(self, n, dtype=torch.float32):
        """A pinned host buffer of >= n elements for an asynchronous D2H copy.  Buffers are recycled only once the
        caller has dropped every array sliced from them (tracked with a weakref), so results stay valid for as long as
        they are referenced and a steady-state loop allocates nothing."""
        for i, (t, ref) in enumerate(self._pinned):
            if t.dtype == dtype and t.numel() >= n and (ref is None or ref() is None):
                return i, t
        t = torch.empty(max(int(n), 1), dtype=dtype).pin_memory()
        self._pinned = [e for e in self._pinned if e[1] is None or e[1]() is not None or e[0].numel() >= n][-7:]
        self._pinned.append((t, None))
        return len(self._pinned) - 1, t

    def _to_host(self, dev_tensor):
        """device tensor -> numpy view of a pinned buffer (async copy on the current stream + one stream sync)."""
        flat = dev_tensor.reshape(-1)
        i, t = self._host_out(flat.numel(), flat.dtype)
        t[:flat.numel()].copy_(flat, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        arr = t.numpy()[:flat.numel()].reshape(tuple(dev_tensor.shape))
        self._pinned[i] = (t, weakref.ref(arr.base if arr.base is not None else arr))
        return arr

    # ---- reference-audio front-end (f3, mel half) -----------------------------------------------------
    def process_audio(self, wav):
        """reference inference/StyleSinger.py:79-92 for a waveform ARRAY already at ``audio_sample_rate`` (decoding and
        resampling a file is librosa's job in the reference and stays outside this package): returns ``(wav, mel)`` with the
        waveform zero-padded / cut to ``len(mel) * hop_size`` samples as float16 and the log10-mel [T, 80] as float32 numpy,
        computed by the CUDA front-end (ssb_melspec_forward)."""
        from .engine import MelSpectrogram
        if isinstance(wav, str):
            raise NotImplementedError("pass the decoded waveform (float array at hparams['audio_sample_rate'])")
        if getattr(self, "_melspec", None) is None:
            self._melspec = MelSpectrogram(self.hparams, self.device)
        wav = np.asarray(wav, dtype=np.float32).reshape(-1)
        mel = self._to_host(self._melspec(wav))
        n = mel.shape[0] * int(self.hparams.get("hop_size", 256))  # utils/audios/__init__.py:71-73 (librosa_pad_lr, then cut)
        out = np.zeros(n, np.float32)
        out[:min(n, len(wav))] = wav[:n]
        return out.astype(np.float16), mel

    def emotion_embed(self, processed_wav, weights=None):
        """`inp['emo_embed'] = Embed_utterance(processed_wav, using_partials=True)` of reference inference/StyleSinger.py:103-106
        on the CUDA front-end (stylesinger_b200.emotion): ``processed_wav`` is the output of the reference's preprocess_wav
        (16 kHz, volume-normalised, VAD-trimmed - librosa / webrtcvad, outside this package); the encoder weights come from
        ``weights`` (path / checkpoint dict / state_dict) or hparams['emotion_encoder_path'] on first use."""
        from . import emotion
        if weights is not None or not emotion.is_loaded():
            emotion.load_model(weights if weights is not None else self.hparams["emotion_encoder_path"], self.device)
        return emotion.embed_utterance(processed_wav, using_partials=True)

    def preprocess_input(self, inp, spk_embed_fn=None, pitch_fn=None, preprocess_wav_fn=None):
        """reference inference/StyleSinger.py:94-137 with the reference-owned arithmetic on the GPU (log-mel of the reference
        audio, emotion embedding) and the third-party models as callables, since their packages are not part of this one:

        * ``inp['ref_audio']``: the decoded reference waveform at hparams['audio_sample_rate'] (the reference passes a path and
          lets librosa decode it);
        * ``spk_embed_fn(wav)`` = ``VoiceEncoder().embed_utterance`` (resemblyzer), or ``inp['spk_embed']`` given;
        * ``preprocess_wav_fn(ref_audio)`` = ``data_gen.tts.emotion.inference.preprocess_wav`` (librosa + webrtcvad) feeding
          ``emotion_embed`` (hparams['emotion_encoder_path']), or ``inp['emo_embed']`` given;
        * ``pitch_fn(wav, sample_rate, time_step_s, f0_min, f0_max, voicing_threshold)`` = the parselmouth ``to_pitch_ac``
          call (:126-129) returning Hz per frame, or ``inp['f0']`` given (already aligned to the mel).

        Fills ``mel``, ``spk_embed``, ``emo_embed``, ``item_name``, ``ph_token``, ``wav_fn``, ``f0`` like the reference."""
        hp = self.hparams
        if self.ph_encoder is None:
            raise ValueError("preprocess_input needs the ph_encoder (utils/text/text_encoder.py build_token_encoder)")
        ph_token = self.ph_encoder.encode(" ".join(inp["ph"]))
        ref_audio = inp["ref_audio"]
        wav, mel = self.process_audio(ref_audio)
        inp["mel"] = mel
        if hp.get("use_spk_id"):  # the speaker is an id of the training set, not an embedding of the reference audio
            if "spk_id" not in inp:
                raise ValueError("inp['spk_id'] required: the model was trained with use_spk_id")
        elif spk_embed_fn is not None:
            inp["spk_embed"] = spk_embed_fn(wav)
        elif "spk_embed" not in inp:
            raise ValueError("spk_embed_fn or inp['spk_embed'] required (resemblyzer VoiceEncoder is third-party)")
        if preprocess_wav_fn is not None:
            inp["emo_embed"] = self.emotion_embed(preprocess_wav_fn(ref_audio))
        elif "emo_embed" not in inp and self.hparams["emo"]:  # a model without emo reads none (StyleSinger.py:44-47)
            raise ValueError("preprocess_wav_fn or inp['emo_embed'] required")
        inp.update({"item_name": inp["name"], "ph_token": ph_token, "wav_fn": ref_audio})
        if pitch_fn is not None:
            time_step = hp["hop_size"] / hp["audio_sample_rate"] * 1000
            f0 = pitch_fn(wav, hp["audio_sample_rate"], time_step / 1000, 80, 800, 0.6)
            inp["f0"] = pad_f0_to_mel(f0, len(mel), hp["hop_size"])
        elif "f0" not in inp:
            raise ValueError("pitch_fn or inp['f0'] required (parselmouth is third-party)")
        return inp

    # ---- reference-compatible single-utterance path ------------------------------------------------
    def input_to_batch(self, item) -> PackedBatch:
        """reference inference/StyleSinger.py:139-170 (B=1 assembly).  ``item['f0']`` is the raw extractor output in Hz
        (0 = unvoiced), exactly what ``preprocess_input`` produces: like the reference (:152) it goes through
        ``norm_interp_f0`` (log2 Hz, unvoiced frames interpolated) before it becomes the style extractor's ``ref_f0``.
        A model without emo reads no ``emo_embed`` (forward_model passes None, :44-47), one without style no ``mel`` /
        ``f0`` (get_style is skipped, stylesinger.py:149-151): the item may then leave them out.  A use_spk_id model reads
        the integer ``item['spk_id']`` instead of ``spk_embed``."""
        hp = self.hparams
        u = {"txt_tokens": torch.as_tensor(item["ph_token"]).long(), "note": torch.as_tensor(item["note"]).long(),
             "note_dur": torch.as_tensor(item["note_dur"]).float(), "note_type": torch.as_tensor(item["note_type"]).long()}
        if hp.get("use_spk_id"):  # the line the reference leaves commented out (inference/StyleSinger.py:146,159)
            u["spk_id"] = int(item["spk_id"])
        else:
            u["spk_embed"] = torch.as_tensor(item["spk_embed"]).float()
        if hp["emo"]:
            u["emo_embed"] = torch.as_tensor(item["emo_embed"]).float()
        if hp["style"]:
            f0, _ = norm_interp_f0(np.asarray(item["f0"]), hp.get("pitch_norm", "log"), hp.get("use_uv", True),
                                   hp.get("f0_mean", 400.0), hp.get("f0_std", 100.0))
            u["ref_mels"] = torch.as_tensor(item["mel"]).float()
            u["ref_f0"] = torch.from_numpy(f0)
        if item.get("mel2ph") is not None:
            u["mel2ph"] = torch.as_tensor(item["mel2ph"]).long()
        return pack_batch([u], use_mel2ph="mel2ph" in u, emo=hp["emo"], style=hp["style"],
                          spk_id=bool(hp.get("use_spk_id")))

    def forward_model(self, inp, seed=0, noise=None, voc_noise=None, return_mel=False):
        """reference inference/StyleSinger.py:41-64: returns the waveform (np.float32 [T*hop]).
        `noise` / `voc_noise` inject the reference's random draws (parity tests); `return_mel` adds the raw mel_out."""
        r = self.infer_packed(self.input_to_batch(inp), seed=seed, noise=noise, voc_noise=voc_noise, return_mel=return_mel)
        return (r[0][0], r[1][0]) if return_mel else r[0]

    # ---- batched path --------------------------------------------------------------------------------
    def infer_batch(self, utts: List[dict], seed=0, use_mel2ph=True, return_mel=False, seeds=None):
        """seeds: one seed per utterance instead of `seed`; utterance b then gets what forward_model(utts[b],
        seed=seeds[b]) gives, whatever else the batch holds (see run_device)."""
        if seeds is not None:  # validated before anything reaches the device
            seeds = utt_seeds(seeds, len(utts))
        return self.infer_packed(self.model.pack_batch(utts, use_mel2ph=use_mel2ph, pin=True), seed=seed, return_mel=return_mel,
                                 seeds=seeds)

    def run_device(self, pb_dev: PackedBatch, seed=0, noise=None, voc_noise=None, seeds=None):
        """Device-resident ph -> mel -> wav: returns (mel [sumF,80] raw model output, f0 [sumF],
        wav [sumF'*hop], frame_offsets of the wav) as device tensors.
        seeds: one Philox seed per utterance (engine.utt_seeds) for the model and the vocoder alike, instead of the
        call's `seed`; it cannot be combined with injected noise."""
        if seeds is not None:
            seeds = utt_seeds(seeds, pb_dev.B)
            if noise or voc_noise:
                raise ValueError("seeds: per-utterance seeds key the in-kernel noise; noise / voc_noise must be None")
        dur = None
        if pb_dev.frame_offsets is None:
            dur, _ = self.model.predict_durations(pb_dev)
            d = dur.cpu().numpy()  # the host needs the frame count (the reference syncs here too)
            po = pb_dev.ph_offsets
            lens = [int(d[po[i]:po[i + 1]].sum()) for i in range(pb_dev.B)]
            pb_dev.frame_offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        out = self.model.forward(pb_dev, noise=noise, seed=seed, dur=dur, want=("mel_out", "f0_denorm"), seeds=seeds)
        mel, f0 = out["mel_out"], out["f0_denorm"]
        fo = pb_dev.frame_offsets
        n = int(fo[-1])
        # inference/StyleSinger.py:56-62: clip to [mel_vmin, mel_vmax]; drop all-zero (padding) frames
        melc = mel.clone()
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        check(lib.ssb_mel_postprocess(C.c_void_p(melc.data_ptr()), n, float(self.hparams["mel_vmin"]),
                                      float(self.hparams["mel_vmax"]), C.c_void_p(self._cnt.data_ptr()), stream),
              "ssb_mel_postprocess")
        fo_v, f0_v = fo, f0
        # Frames whose mel is exactly zero only exist where an explicit mel2ph carries zeros (padding frames):
        # pack_batch records that on the host, so the common case needs no device->host sync between model and vocoder.
        if pb_dev.may_have_pad_frames and int(self._cnt.item()) != n:  # rare: compact on the host side
            keep = (mel.abs().sum(-1) > 0)
            k = keep.cpu().numpy()
            lens = [int(k[fo[i]:fo[i + 1]].sum()) for i in range(pb_dev.B)]
            fo_v = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
            melc, f0_v = melc[keep].contiguous(), f0[keep].contiguous()
        vn = voc_noise or {}
        wav = self.vocoder.generate(melc, f0_v if self.hparams.get("use_nsf") else None, fo_v,
                                    rand_ini=vn.get("rand_ini"), src_noise=vn.get("src_noise"), seed=seed, seeds=seeds)
        return mel, f0, wav, fo_v

    def infer_packed(self, pb: PackedBatch, seed=0, return_mel=False, noise=None, voc_noise=None, seeds=None):
        """Host buffers in, host buffers out (H2D of the inputs, D2H of the waveform)."""
        if seeds is not None:  # validated before anything reaches the device
            seeds = utt_seeds(seeds, pb.B)
        pb_dev = pb.to(self.device)
        mel, f0, wav, fo_v = self.run_device(pb_dev, seed=seed, noise=noise, voc_noise=voc_noise, seeds=seeds)
        wav_h = self._to_host(wav)
        hop = self.vocoder.hop
        wavs = [wav_h[fo_v[i] * hop:fo_v[i + 1] * hop] for i in range(pb_dev.B)]
        if return_mel:
            mel_h = self._to_host(mel)
            fo = pb_dev.frame_offsets
            return wavs, [mel_h[fo[i]:fo[i + 1]] for i in range(pb_dev.B)]
        return wavs
