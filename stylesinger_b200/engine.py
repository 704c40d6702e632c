"""Host-side engine: checkpoint packing, ragged batches, workspaces and the calls into the C ABI.

PyTorch is used here only for device memory, streams and host<->device copies; every arithmetic
operation of the path runs in libstylesinger_b200.so (see include/stylesinger_b200.h).
"""
import ctypes as C
import math
import operator
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np
import torch

from . import _lib
from ._lib import AcousticInputs, AcousticOutputs, HParams, ModelSwitches, TensorDesc, VocoderConfigEx, check, lib
from .hparams import DEFAULT_VOCODER_CONFIG, TC_PRECISIONS, resolve, switches
from .schedules import multinomial_table, prodiff_table, sampler_table

MEL_DECODERS = {"diffsinger": 0, "prodiff": 1, "fft": 2}  # SSB_MEL_DECODER_* of include/stylesinger_b200.h
F0_GENS = {"gmdiff": 0, "conv": 1}  # SSB_F0_GEN_*


def _require_cuda():
    if not torch.cuda.is_available():
        raise _lib.SsbError("stylesinger_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")


def _ptr(t: Optional[torch.Tensor]):
    """Device pointer of a tensor handed to the C ABI. The library reads plain row-major memory, so a strided
    (e.g. transposed / Fortran-ordered) view would be silently misread: refuse it loudly."""
    if t is None:
        return None
    if not t.is_contiguous():
        raise ValueError("stylesinger_b200: tensors passed to the C ABI must be contiguous (call .contiguous())")
    return C.c_void_p(t.data_ptr())


def utt_seeds(seeds, B) -> np.ndarray:
    """One Philox seed per utterance -> host uint64 [B].  Each utterance then draws exactly the noise of a B = 1 call
    with its seed, whatever batch it runs in (csrc/philox.cuh).  Raises ValueError for a length other than B or a seed
    outside [0, 2**64), TypeError for a seed that is not an integer."""
    s = [operator.index(v) for v in seeds]
    if len(s) != B:
        raise ValueError(f"seeds: expected one seed per utterance ({B}), got {len(s)}")
    bad = [v for v in s if not 0 <= v < 2 ** 64]
    if bad:
        raise ValueError(f"seeds: every seed must be in [0, 2**64), got {bad[0]}")
    return np.array(s, dtype=np.uint64)


def _descs(named: Dict[str, torch.Tensor]):
    """ssb_tensor_desc array over fp32 contiguous CPU copies (kept alive by the returned list)."""
    keep, arr = [], (TensorDesc * len(named))()
    for i, (k, v) in enumerate(named.items()):
        t = v.detach().to("cpu", torch.float32).contiguous()
        if t.dim() == 0:
            t = t.reshape(1)
        if t.dim() > 4:
            raise ValueError(f"{k}: rank > 4")
        keep.append(t)
        kb = k.encode()
        keep.append(kb)
        arr[i].name = kb
        arr[i].data = t.data_ptr()
        arr[i].ndim = t.dim()
        for d in range(t.dim()):
            arr[i].shape[d] = t.shape[d]
    return arr, keep


def sinusoid_table(n, dim=256, padding_idx=0):
    """SinusoidalPositionalEmbedding.get_embedding (reference modules/commons/common_layers.py:111-127),
    computed on the host exactly like the reference does at module construction."""
    half = dim // 2
    e = math.log(10000) / (half - 1)
    e = torch.exp(torch.arange(half, dtype=torch.float) * -e)
    e = torch.arange(n, dtype=torch.float).unsqueeze(1) * e.unsqueeze(0)
    e = torch.cat([torch.sin(e), torch.cos(e)], dim=1).view(n, -1)
    e[padding_idx, :] = 0
    return e


def step_embedding(T, C_):
    """SinusoidalPosEmb(t) for t = 0..T-1 (reference modules/diff/net.py:31-44)."""
    half = C_ // 2
    e = math.log(10000) / (half - 1)
    e = torch.exp(torch.arange(half) * -e)
    e = torch.arange(T)[:, None] * e[None, :]
    return torch.cat((e.sin(), e.cos()), dim=-1).float().contiguous()


@dataclass
class PackedBatch:
    """A ragged batch in the library's tight layout. Offsets are host int32 arrays [B+1]."""
    B: int
    ph_offsets: np.ndarray
    ref_offsets: Optional[np.ndarray]  # None for a model without style (no reference mels)
    frame_offsets: Optional[np.ndarray]
    t: Dict[str, torch.Tensor] = field(default_factory=dict)  # txt_tokens, note, note_type (int32), note_dur,
    # [spk_embed], [emo_embed], [ref_mels, ref_f0], [mel2ph int32], [f0], [uv]
    may_have_pad_frames: bool = True  # False when the host knows every frame maps to a phone (mel2ph > 0 everywhere)
    spk_ids: Optional[np.ndarray] = None  # host int32 [B] speaker ids, for a use_spk_id model (in place of t["spk_embed"])

    def to(self, device, non_blocking=True):
        return PackedBatch(self.B, self.ph_offsets, self.ref_offsets, self.frame_offsets,
                           {k: v.to(device, non_blocking=non_blocking) for k, v in self.t.items()},
                           self.may_have_pad_frames, self.spk_ids)

    def h2d_bytes(self):
        return int(sum(v.numel() * v.element_size() for v in self.t.values()))

    @property
    def total_frames(self):
        return int(self.frame_offsets[-1]) if self.frame_offsets is not None else 0


def pack_batch(utts: List[dict], use_mel2ph=True, pin=False, emo=True, style=True, spk_id=False) -> PackedBatch:
    """Concatenate per-utterance CPU tensors (as produced by synth.make_utterance) into one PackedBatch.
    emo / style: the model switches of the model the batch is for.  Without emo, no emo_embed is packed (utterances need
    none); without style, no ref_mels / ref_f0 are packed and ref_offsets is None.  spk_id: the batch is for a use_spk_id
    model: each utterance's integer u["spk_id"] goes to the host array spk_ids, and no spk_embed is packed."""
    def offs(lens):
        return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)

    B = len(utts)
    po = offs([len(u["txt_tokens"]) for u in utts])
    ro = offs([u["ref_mels"].shape[0] for u in utts]) if style else None
    fo = offs([len(u["mel2ph"]) for u in utts]) if use_mel2ph else None
    cat = lambda k, dt: torch.cat([u[k].reshape(-1) if u[k].dim() == 1 else u[k] for u in utts]).to(dt).contiguous()
    t = {"txt_tokens": cat("txt_tokens", torch.int32), "note": cat("note", torch.int32),
         "note_type": cat("note_type", torch.int32), "note_dur": cat("note_dur", torch.float32)}
    ids = None
    if spk_id:
        ids = np.array([operator.index(u["spk_id"]) for u in utts], dtype=np.int32)
    else:
        t["spk_embed"] = torch.stack([u["spk_embed"] for u in utts]).float().contiguous()
    if emo:
        t["emo_embed"] = torch.stack([u["emo_embed"] for u in utts]).float().contiguous()
    if style:
        t["ref_mels"] = cat("ref_mels", torch.float32)
        t["ref_f0"] = cat("ref_f0", torch.float32)
    pad = False  # predicted durations: the length regulator never emits a zero entry inside an utterance
    if use_mel2ph:
        t["mel2ph"] = cat("mel2ph", torch.int32)
        pad = bool((t["mel2ph"] <= 0).any())
    if pin and torch.cuda.is_available():
        t = {k: v.pin_memory() for k, v in t.items()}
    return PackedBatch(B, po, ro, fo, t, pad, ids)


class _Workspace:
    def __init__(self, device):
        self.device = device
        self.buf = None

    def get(self, nbytes):
        if self.buf is None or self.buf.numel() < nbytes:
            self.buf = None
            self.buf = torch.empty(int(nbytes * 1.05) + 4096, dtype=torch.uint8, device=self.device)
        return self.buf


class AcousticModel:
    """Packed StyleSinger acoustic model on one GPU (ssb_model_t).  hparams['decoder'] selects the mel decoder:
    'diffsinger' (FFT decoder + DDPM refinement, the default) or 'prodiff' (the ProDiff teacher, decoder_inp -> mel).
    hparams['f0_gen'] selects the F0 generator: 'gmdiff' (two F0 diffusion samplers, the default) or 'conv' (two
    deterministic FastSpeech-2 PitchPredictors; no F0 schedule, no F0 noise).  The model switches hparams['emo'],
    ['style'], ['umln'] and ['use_txt_cond'] (all True by default) select the modules the checkpoint has
    (ssb_model_create_ex3); batches for a model without emo / style need no emo_embed / reference mels
    (pack_batch(..., emo=, style=), or ``self.pack_batch``).  hparams['decoder'] 'fft' is the FastSpeech 2 decoder alone:
    its mel is the output, with no diffusion.  hparams['use_spk_id'] makes spk_embed_proj a speaker table looked up by
    integer ids (utterances carry ``spk_id`` instead of ``spk_embed``; ssb_model_create_ex4).  Both need
    hparams['extended_models'] = True.  hparams['tc_precision'] ('split' or 'fp16') sets the
    precision of the mel DiffNet's tensor-core GEMMs (set_mel_precision)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], hparams=None, device=None, max_positions=4096):
        _require_cuda()
        self.hp = resolve(hparams)
        self.device = torch.device(device if device is not None else "cuda:0")
        torch.cuda.set_device(self.device)
        sd = {k: v for k, v in state_dict.items() if isinstance(v, torch.Tensor)}
        sd = dict(sd)
        sd["__pos_table"] = sinusoid_table(max_positions, self.hp["hidden_size"])
        if "encoder.embed_tokens.weight" not in sd and "encoder_embed_tokens.weight" in sd:
            sd["encoder.embed_tokens.weight"] = sd["encoder_embed_tokens.weight"]
        hp = self.hp
        h = HParams(hp["hidden_size"], hp["enc_layers"], hp["dec_layers"], hp["enc_ffn_kernel_size"],
                    hp["dec_ffn_kernel_size"], hp["dur_predictor_layers"], hp["dur_predictor_kernel"],
                    int(sd["encoder.embed_tokens.weight"].shape[0]), hp["nRQ"], hp["rq_depth"],
                    hp["residual_channels"], hp["residual_layers"], hp["dilation_cycle_length"],
                    hp["f0_residual_channels"], hp["f0_residual_layers"], hp["f0_dilation_cycle_length"],
                    hp["audio_num_mel_bins"])
        self.mel_decoder = hp["decoder"]
        self.f0_gen = hp["f0_gen"]
        self.switches = switches(hp)
        self.spk_id = bool(hp["use_spk_id"])
        if self.spk_id and hp.get("num_spk") is not None:  # Embedding(num_spk + 1, H) (fs2.py:37-38)
            rows = int(sd["spk_embed_proj.weight"].shape[0])
            if rows != int(hp["num_spk"]) + 1:
                raise ValueError(f"spk_embed_proj.weight has {rows} rows; hparams num_spk = {hp['num_spk']} needs "
                                 f"num_spk + 1 = {int(hp['num_spk']) + 1}")
        sw = ModelSwitches(**{k: int(v) for k, v in self.switches.items()})
        arr, keep = _descs(sd)
        handle = C.c_void_p()
        check(lib.ssb_model_create_ex4(C.byref(handle), arr, len(sd), C.byref(h), MEL_DECODERS[self.mel_decoder],
                                       F0_GENS[self.f0_gen], C.byref(sw), int(self.spk_id)), "ssb_model_create_ex4")
        self._h = handle
        self._ws = _Workspace(self.device)
        self.T = self.f0_T = None
        # an FFT model has no mel sampler, a conv-F0 model no F0 samplers: neither gets a schedule
        self.set_timesteps(hp["timesteps"] if self.mel_decoder != "fft" else None,
                           hp["f0_timesteps"] if self.f0_gen == "gmdiff" else None)
        self.K = None  # K_step of the mel sampler; None follows T
        if self.mel_decoder == "diffsinger" and int(hp["K_step"]) != hp["timesteps"]:
            self.set_mel_k_step(int(hp["K_step"]))
        self.set_mel_precision(hp["tc_precision"])

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            lib.ssb_model_free(h)
            self._h = None

    def pack_batch(self, utts: List[dict], use_mel2ph=True, pin=False) -> PackedBatch:
        """pack_batch with the fields this model reads (no emo_embed without emo, no reference mels without style, speaker
        ids instead of spk_embed with use_spk_id)."""
        return pack_batch(utts, use_mel2ph, pin, emo=self.switches["emo"], style=self.switches["style"], spk_id=self.spk_id)

    def set_tensor_cores(self, enable=True):
        """wgmma (fp16 hi/lo split, 3 MMAs) vs fp32 FFMA for the denoiser layer GEMMs. Returns the mode in effect."""
        return bool(lib.ssb_model_set_tensor_cores(self._h, 1 if enable else 0))

    def set_persistent(self, enable=True):
        """Single-launch persistent sampler kernel for small batches (True) vs one launch per GEMM (False)."""
        return bool(lib.ssb_model_set_persistent(self._h, 1 if enable else 0))

    def set_persistent_groups(self, enable=True):
        """Large batches: run the mel sampler as one persistent launch per group of <= 48 row tiles (default off)."""
        return bool(lib.ssb_model_set_persistent_groups(self._h, 1 if enable else 0))

    def set_mel_precision(self, mode: str):
        """Precision of the mel DiffNet's tensor-core GEMMs on every mel sampler (DDPM, K_step, PLMS, ProDiff): 'split'
        (fp16 hi/lo planes, 3 MMAs per K step; the default) or 'fp16' (one MMA on operands rounded once to fp16, faster, at
        the accuracy cost stated in the README).  The F0 samplers and every other module stay split; GEMMs on the FFMA
        path are unchanged.  An unknown mode raises ValueError and changes nothing."""
        if mode not in TC_PRECISIONS:
            raise ValueError(f"mel precision must be one of {sorted(TC_PRECISIONS)}, got {mode!r}")
        check(lib.ssb_model_set_mel_precision(self._h, TC_PRECISIONS[mode]), "ssb_model_set_mel_precision")
        self.mel_precision = mode

    def set_fft_tensor_cores(self, enable: bool) -> bool:
        """Decoder FFT-block FFN GEMMs on the tensor-core kernel for batches of >= 1024 frames (default on)."""
        return bool(lib.ssb_model_set_fft_tensor_cores(self._h, 1 if enable else 0))

    # -- schedules -------------------------------------------------------------------------------
    def set_timesteps(self, T=None, f0_T=None):
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        if T is not None and T != self.T:
            emb = step_embedding(T, self.hp["residual_channels"])
            if self.mel_decoder == "prodiff":
                g = np.ascontiguousarray(prodiff_table(T, self.hp["schedule_type"]))
            else:
                g = np.ascontiguousarray(sampler_table(T, self.hp["max_beta"]))
            check(lib.ssb_model_set_schedule(self._h, 0, T, C.c_void_p(emb.data_ptr()), g.ctypes.data_as(C.c_void_p),
                                             None, stream), "ssb_model_set_schedule(mel)")
            self.T = T
        if f0_T is not None and f0_T != self.f0_T:  # (the library refuses it on an f0_gen 'conv' model)
            emb = step_embedding(f0_T, self.hp["f0_residual_channels"])
            g = np.ascontiguousarray(sampler_table(f0_T, self.hp["f0_max_beta"]))
            m = np.ascontiguousarray(multinomial_table(f0_T, self.hp["f0_max_beta"]))
            check(lib.ssb_model_set_schedule(self._h, 1, f0_T, C.c_void_p(emb.data_ptr()),
                                             g.ctypes.data_as(C.c_void_p), m.ctypes.data_as(C.c_void_p), stream),
                  "ssb_model_set_schedule(f0)")
            self.f0_T = f0_T

    def set_mel_k_step(self, K=None):
        """hparams['K_step'] of the DiffSinger mel sampler (shallow diffusion): q_sample at K-1 of the T-step schedule, then
        K reverse steps; injected mel noise is then [(K+1), sumF, 80].  None or 0 follows T.  A K above T fails at the
        sampler call; any K on a 'prodiff' model fails here."""
        K = int(K or 0)
        check(lib.ssb_model_set_mel_k_step(self._h, K), "ssb_model_set_mel_k_step")
        self.K = K or None

    # -- helpers ---------------------------------------------------------------------------------
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _inputs(self, pb: PackedBatch, noise=None, seed=0, skip_mel=False, dur=None, f0=None, uv=None):
        a = AcousticInputs()
        a.B = pb.B
        self._keep = [np.ascontiguousarray(pb.ph_offsets, np.int32)]
        a.ph_offsets = self._keep[0].ctypes.data
        if self.switches["style"]:  # a model without style reads no reference offsets, mels or f0
            self._keep.append(np.ascontiguousarray(pb.ref_offsets, np.int32))
            a.ref_offsets = self._keep[-1].ctypes.data
        if pb.frame_offsets is not None:
            fo = np.ascontiguousarray(pb.frame_offsets, np.int32)
            self._keep.append(fo)
            a.frame_offsets = fo.ctypes.data
        t = pb.t
        keys = ["txt_tokens", "note", "note_type", "note_dur"]
        if self.spk_id:  # the library reads the host ids (a batch without them reaches it as NULL and is refused)
            if pb.spk_ids is not None:
                self._keep.append(np.ascontiguousarray(pb.spk_ids, np.int32))
                a.spk_ids = self._keep[-1].ctypes.data
        else:
            keys.append("spk_embed")
        keys += ["emo_embed"] if self.switches["emo"] else []  # forward_model passes none then (inference/StyleSinger.py:44-47)
        keys += ["ref_mels", "ref_f0"] if self.switches["style"] else []
        for k in keys:
            assert t[k].is_cuda and t[k].is_contiguous(), k
            setattr(a, k, t[k].data_ptr())
        if "mel2ph" in t and dur is None:
            a.mel2ph = t["mel2ph"].data_ptr()
        if dur is not None:
            a.dur = dur.data_ptr()
        f0 = f0 if f0 is not None else t.get("f0")
        uv = uv if uv is not None else t.get("uv")
        if f0 is not None:
            a.f0 = f0.data_ptr()
            if uv is not None:
                a.uv = uv.data_ptr()
        if noise:
            for i in range(2):
                if noise.get("f0_gauss") is not None:
                    a.f0_gauss_noise[i] = noise["f0_gauss"][i].data_ptr()
                    a.f0_unif_noise[i] = noise["f0_unif"][i].data_ptr()
            if noise.get("mel") is not None:
                a.mel_noise = noise["mel"].data_ptr()
        a.seed = int(seed)
        a.skip_mel_diffusion = 1 if skip_mel else 0
        # reference hparam: 0 / absent = DDPM (the StyleSinger default); the ProDiff sampler ignores it, as the reference does
        # (an FFT model has no sampler at all)
        a.pndm_speedup = 0 if self.mel_decoder != "diffsinger" else int(self.hp.get("pndm_speedup") or 0)
        return a

    # -- entry points ------------------------------------------------------------------------------
    def predict_durations(self, pb: PackedBatch):
        """DurationPredictor.inference; returns (dur int32 [sumP], log-dur f32 [sumP]) on the device."""
        a = self._inputs(pb)
        n = lib.ssb_durations_workspace_bytes(self._h, C.byref(a))
        if n == 0:
            check(-1, "ssb_durations_workspace_bytes")
        ws = self._ws.get(n)
        P = int(pb.ph_offsets[-1])
        dur = torch.empty(P, dtype=torch.int32, device=self.device)
        logdur = torch.empty(P, dtype=torch.float32, device=self.device)
        check(lib.ssb_predict_durations(self._h, C.byref(a), _ptr(dur), _ptr(logdur), _ptr(ws), ws.numel(), self._stream()),
              "ssb_predict_durations")
        return dur, logdur

    def forward(self, pb: PackedBatch, noise=None, seed=0, skip_mel_diffusion=False, dur=None,
                want=("mel_out", "f0_denorm"), seeds=None):
        """StyleSinger.forward(infer=True). `pb` must carry frame_offsets (+ mel2ph, or pass `dur`).
        Returns a dict of tight device tensors for the keys in `want`.
        seeds: one seed per utterance (see utt_seeds) instead of `seed`: utterance b then gets the outputs of a B = 1
        forward with seed=seeds[b].  Injected noise cannot be combined with it."""
        assert pb.frame_offsets is not None, "frame_offsets required (run predict_durations first)"
        keys = None
        if seeds is not None:
            keys = utt_seeds(seeds, pb.B)
            if noise and any(v is not None for v in noise.values()):
                raise ValueError("seeds: per-utterance seeds key the in-kernel noise; injected noise must be None")
        a = self._inputs(pb, noise, seed, skip_mel_diffusion, dur)
        Fs, Ps = int(pb.frame_offsets[-1]), int(pb.ph_offsets[-1])
        Rs = int(pb.ref_offsets[-1]) if pb.ref_offsets is not None else 0
        shapes = {"mel_out": (Fs, 80), "f0_denorm": (Fs,), "encoder_out": (Ps, 256), "style": (Fs, 256),
                  "rq_codes": (Rs, self.hp["rq_depth"]), "pitch_pred": (Fs, 2), "decoder_inp": (Fs, 256),
                  "coarse_mel": (Fs, 80), "diff_cond": (Fs, 256), "mel2ph": (Fs,), "spk_proj": (pb.B, 256),
                  "emo_proj": (pb.B, 256)}
        o = AcousticOutputs()
        out = {}
        want = set(want)
        # outputs of switched-off modules do not exist (the library refuses them too; a style-off batch has no reference
        # rows, so an empty rq_codes buffer would otherwise reach it as NULL)
        for k, sw in (("emo_proj", "emo"), ("style", "style"), ("rq_codes", "style")):
            if k in want and not self.switches[sw]:
                raise _lib.SsbError(f"AcousticModel.forward: a model without {sw} (hparams {sw}=False) has no {k}")
        if "diff_cond" in want and self.mel_decoder == "fft":
            raise _lib.SsbError("AcousticModel.forward: a model with decoder 'fft' has no diff_cond (there is no ln_proj)")
        if skip_mel_diffusion:
            want.discard("mel_out")  # never written in that mode: do not hand back an uninitialised buffer
        else:
            want.add("mel_out")
        for k in want:
            dt = torch.int32 if k in ("rq_codes", "mel2ph") else torch.float32
            out[k] = torch.empty(shapes[k], dtype=dt, device=self.device)
            setattr(o, k, out[k].data_ptr())
        n = lib.ssb_acoustic_workspace_bytes(self._h, C.byref(a))
        if n == 0:
            check(-1, "ssb_acoustic_workspace_bytes")
        ws = self._ws.get(n)
        if keys is None:
            check(lib.ssb_acoustic_forward(self._h, C.byref(a), C.byref(o), _ptr(ws), ws.numel(), self._stream()),
                  "ssb_acoustic_forward")
        else:
            check(lib.ssb_acoustic_forward_keyed(self._h, C.byref(a), keys.ctypes.data, C.byref(o), _ptr(ws), ws.numel(),
                                                 self._stream()), "ssb_acoustic_forward_keyed")
        return out

    def mel_diffusion(self, cond, coarse, frame_offsets, noise=None, seed=0):
        """DiffusionDecoder.forward(infer=True): cond [sumF,256], coarse [sumF,80] -> mel [sumF,80].  noise: [(K+1), sumF, 80]
        (the q_sample draw, then one per step t = K-1 .. 0; K = K_step, else T), or None for the in-kernel Philox."""
        fo = np.ascontiguousarray(frame_offsets, np.int32)
        B = len(fo) - 1
        n = lib.ssb_mel_diffusion_workspace_bytes(self._h, fo.ctypes.data, B)
        if n == 0:
            check(-1, "ssb_mel_diffusion_workspace_bytes")
        ws = self._ws.get(n)
        mel = torch.empty((int(fo[-1]), 80), dtype=torch.float32, device=self.device)
        check(lib.ssb_mel_diffusion_sample(self._h, _ptr(cond), _ptr(coarse), fo.ctypes.data, B, _ptr(noise), int(seed),
                                           _ptr(mel), _ptr(ws), ws.numel(), self._stream()), "ssb_mel_diffusion_sample")
        return mel

    def mel_prodiff(self, cond, frame_offsets, noise=None, seed=0):
        """ProDiffusion.forward(cond, infer=True) on a 'prodiff' model: cond = decoder_inp [sumF,256] (device, tight) ->
        mel [sumF,80].  noise: [(T+1), sumF, 80] (the x_T draw, then one per step), or None for the in-kernel Philox."""
        fo = np.ascontiguousarray(frame_offsets, np.int32)
        B = len(fo) - 1
        n = lib.ssb_mel_prodiff_workspace_bytes(self._h, fo.ctypes.data, B)
        if n == 0:
            check(-1, "ssb_mel_prodiff_workspace_bytes")
        ws = self._ws.get(n)
        mel = torch.empty((int(fo[-1]), 80), dtype=torch.float32, device=self.device)
        check(lib.ssb_mel_prodiff_sample(self._h, _ptr(cond), fo.ctypes.data, B, _ptr(noise), int(seed), _ptr(mel), _ptr(ws),
                                         ws.numel(), self._stream()), "ssb_mel_prodiff_sample")
        return mel

    def mel_diffusion_plms(self, cond, coarse, frame_offsets, interval, q_noise=None, seed=0):
        """PLMS sampler (hparams['pndm_speedup'] = interval, in [1, K)) over the mel denoiser: K / interval (+1) evaluations."""
        fo = np.ascontiguousarray(frame_offsets, np.int32)
        B = len(fo) - 1
        n = lib.ssb_mel_diffusion_plms_workspace_bytes(self._h, fo.ctypes.data, B)
        if n == 0:
            check(-1, "ssb_mel_diffusion_plms_workspace_bytes")
        ws = self._ws.get(n)
        mel = torch.empty((int(fo[-1]), 80), dtype=torch.float32, device=self.device)
        check(lib.ssb_mel_diffusion_sample_plms(self._h, _ptr(cond), _ptr(coarse), fo.ctypes.data, B, _ptr(q_noise), int(seed),
                                                int(interval), _ptr(mel), _ptr(ws), ws.numel(), self._stream()),
              "ssb_mel_diffusion_sample_plms")
        return mel

    def denoiser_eval(self, which, x, uv, t, cond, frame_offsets):
        fo = np.ascontiguousarray(frame_offsets, np.int32)
        B, Fs = len(fo) - 1, int(fo[-1])
        C_ = self.hp["residual_channels"] if which == 0 else self.hp["f0_residual_channels"]
        L_ = self.hp["residual_layers"] if which == 0 else self.hp["f0_residual_layers"]
        rows = Fs + 16 * (B + 1) + 512
        ws = self._ws.get(rows * (12 * C_ + 2 * C_ * L_ + 1024) * 4 + (1 << 20))
        out = torch.empty((Fs, 80 if which == 0 else 3), dtype=torch.float32, device=self.device)
        check(lib.ssb_denoiser_eval(self._h, which, _ptr(x), _ptr(uv), int(t), _ptr(cond), fo.ctypes.data, B, _ptr(out),
                                    _ptr(ws), ws.numel(), self._stream()), "ssb_denoiser_eval")
        return out

    def f0_diffusion(self, which, cond, lo, hi, frame_offsets, gauss_noise=None, unif_noise=None, seed=0):
        fo = np.ascontiguousarray(frame_offsets, np.int32)
        B, Fs = len(fo) - 1, int(fo[-1])
        C_, L_ = self.hp["f0_residual_channels"], self.hp["f0_residual_layers"]
        rows = Fs + 16 * (B + 1) + 512
        ws = self._ws.get(rows * (12 * C_ + 2 * C_ * L_ + 1024) * 4 + (1 << 20))
        z = torch.empty(Fs, dtype=torch.float32, device=self.device)
        uv = torch.empty(Fs, dtype=torch.int32, device=self.device)
        check(lib.ssb_f0_diffusion_sample(self._h, which, _ptr(cond), _ptr(lo), _ptr(hi), fo.ctypes.data, B,
                                          _ptr(gauss_noise), _ptr(unif_noise), int(seed), _ptr(z), _ptr(uv), _ptr(ws),
                                          ws.numel(), self._stream()), "ssb_f0_diffusion_sample")
        return z, uv

    def pitch_predictor(self, which, x, frame_offsets):
        """PitchPredictor.forward on an f0_gen 'conv' model: which 0 = pitch_predictor (domain agnostic input), 1 =
        pitch_inpainter_predictor (domain specific input); x [sumF,256] (device, tight) -> [sumF,2] (log2-Hz f0, uv
        logit)."""
        fo = np.ascontiguousarray(frame_offsets, np.int32)
        B = len(fo) - 1
        n = lib.ssb_pitch_predictor_workspace_bytes(self._h, fo.ctypes.data, B)
        if n == 0:
            check(-1, "ssb_pitch_predictor_workspace_bytes")
        ws = self._ws.get(n)
        out = torch.empty((int(fo[-1]), 2), dtype=torch.float32, device=self.device)
        check(lib.ssb_pitch_predictor(self._h, int(which), _ptr(x), fo.ctypes.data, B, _ptr(out), _ptr(ws), ws.numel(),
                                      self._stream()), "ssb_pitch_predictor")
        return out

    def fft_encoder(self, txt_tokens, ph_offsets):
        """FastspeechEncoder.forward: int32 tokens [sumP] (device) -> [sumP,256]."""
        po = np.ascontiguousarray(ph_offsets, np.int32)
        B = len(po) - 1
        n = lib.ssb_fft_workspace_bytes(self._h, 0, po.ctypes.data, B)
        if n == 0:
            check(-1, "ssb_fft_workspace_bytes")
        ws = self._ws.get(n)
        out = torch.empty((int(po[-1]), 256), dtype=torch.float32, device=self.device)
        check(lib.ssb_fft_encoder(self._h, _ptr(txt_tokens), po.ctypes.data, B, _ptr(out), _ptr(ws), ws.numel(), self._stream()),
              "ssb_fft_encoder")
        return out

    def fft_decoder(self, x, frame_offsets):
        """FastspeechDecoder.forward: x [sumF,256] (device) -> [sumF,256]."""
        fo = np.ascontiguousarray(frame_offsets, np.int32)
        B = len(fo) - 1
        n = lib.ssb_fft_workspace_bytes(self._h, 1, fo.ctypes.data, B)
        if n == 0:
            check(-1, "ssb_fft_workspace_bytes")
        ws = self._ws.get(n)
        out = torch.empty((int(fo[-1]), 256), dtype=torch.float32, device=self.device)
        check(lib.ssb_fft_decoder(self._h, _ptr(x), fo.ctypes.data, B, _ptr(out), _ptr(ws), ws.numel(), self._stream()),
              "ssb_fft_decoder")
        return out

    def get_style(self, decoder_inp, frame_offsets, ref_mels, ref_f0, ref_offsets):
        """StyleSinger.get_style: (decoder_inp [sumF,256], ref_mels [sumR,80], ref_f0 [sumR]) -> (style [sumF,256], codes)."""
        fo = np.ascontiguousarray(frame_offsets, np.int32)
        ro = np.ascontiguousarray(ref_offsets, np.int32)
        B = len(fo) - 1
        n = lib.ssb_get_style_workspace_bytes(self._h, fo.ctypes.data, ro.ctypes.data, B)
        if n == 0:
            check(-1, "ssb_get_style_workspace_bytes")
        ws = self._ws.get(n)
        style = torch.empty((int(fo[-1]), 256), dtype=torch.float32, device=self.device)
        codes = torch.empty((int(ro[-1]), self.hp["rq_depth"]), dtype=torch.int32, device=self.device)
        check(lib.ssb_get_style(self._h, _ptr(decoder_inp), fo.ctypes.data, _ptr(ref_mels), _ptr(ref_f0), ro.ctypes.data, B,
                                _ptr(style), _ptr(codes), _ptr(ws), ws.numel(), self._stream()), "ssb_get_style")
        return style, codes

    def rvq(self, x, ref_offsets):
        ro = np.ascontiguousarray(ref_offsets, np.int32)
        B, Rs = len(ro) - 1, int(ro[-1])
        D = self.hp["rq_depth"]
        ws = self._ws.get((Rs + 16 * (B + 1) + 512) * (512 + D + 8) * 4 + (1 << 20))
        q = torch.empty((Rs, 256), dtype=torch.float32, device=self.device)
        codes = torch.empty((Rs, D), dtype=torch.int32, device=self.device)
        check(lib.ssb_rvq_lookup(self._h, _ptr(x), ro.ctypes.data, B, _ptr(q), _ptr(codes), _ptr(ws), ws.numel(),
                                 self._stream()), "ssb_rvq_lookup")
        return q, codes


def vocoder_config_ex(h):
    """The generator config keys HifiGanGenerator.__init__ reads (modules/hifigan/hifigan_nsf.py:104-142) -> the C struct.
    ``resblock`` '1' builds ResBlock1 and '2' ResBlock2 (:115; an int is read as its string).  Like the reference's modules,
    ResBlock1 reads the first 3 entries of each dilation list and ResBlock2 the first 2; a shorter list, which the
    reference cannot build either, is refused."""
    rb = str(h.get("resblock", "1"))
    if rb not in ("1", "2"):
        raise ValueError(f"resblock must be '1' (ResBlock1) or '2' (ResBlock2), got {h.get('resblock')!r}")
    nd = 3 if rb == "1" else 2
    ks, ds = h["resblock_kernel_sizes"], h["resblock_dilation_sizes"]
    if len(ds) < len(ks):
        raise ValueError(f"resblock_dilation_sizes has {len(ds)} lists for {len(ks)} resblock kernel sizes")
    vc = VocoderConfigEx()
    vc.n_up = len(h["upsample_rates"])
    if not (1 <= vc.n_up <= 8 and 1 <= len(ks) <= 4):
        raise ValueError("1-8 upsampling stages and 1-4 resblock kernel sizes are supported")
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        vc.up_rates[i], vc.up_kernels[i] = u, k
    vc.initial_channel = h["upsample_initial_channel"]
    vc.n_res = len(ks)
    for j, (k, d) in enumerate(zip(ks, ds)):
        if len(d) < nd:
            raise ValueError(f"ResBlock{rb} reads {nd} dilations per block; resblock_dilation_sizes[{j}] = {list(d)}")
        vc.res_kernels[j] = k
        for m in range(nd):
            vc.res_dilations[j][m] = d[m]
    vc.use_pitch_embed = 1 if h.get("use_pitch_embed") else 0
    vc.sample_rate = h.get("audio_sample_rate", 48000)
    vc.resblock = int(rb)
    return vc


class Vocoder:
    """Packed HiFi-GAN(-NSF) generator on one GPU (ssb_vocoder_t).  ``denoise_c`` > 0 runs the reference's output denoiser
    (hparams['vocoder_denoise_c'], tasks/tts/vocoder_infer/hifigan_nsf.py:73-74) on every generated waveform, with the
    fft_size / hop_size / win_size of ``denoise_hp`` (the reference reads its global hparams; default: ``config``, then the
    WavDenoiser defaults).  Nothing is created for the denoiser unless a call asks for it.  ``tc_precision`` ('split' or
    'fp16', hparams['tc_precision']) sets the precision of the tensor-core GEMMs (set_precision)."""

    def __init__(self, state_dict, config=None, device=None, denoise_c=0.0, denoise_hp=None, tc_precision="split"):
        _require_cuda()
        self.denoise_c = float(denoise_c)
        self._denoise_hp = denoise_hp
        self._denoiser = None
        self.cfg = dict(DEFAULT_VOCODER_CONFIG, **(config or {}))
        self.device = torch.device(device if device is not None else "cuda:0")
        torch.cuda.set_device(self.device)
        h = self.cfg
        vc = vocoder_config_ex(h)
        self.hop = int(np.prod(h["upsample_rates"]))
        sd = {k: v for k, v in state_dict.items() if isinstance(v, torch.Tensor)}
        arr, keep = _descs(sd)
        handle = C.c_void_p()
        check(lib.ssb_vocoder_create_ex(C.byref(handle), arr, len(sd), C.byref(vc)), "ssb_vocoder_create_ex")
        self._h = handle
        self._ws = _Workspace(self.device)
        self.set_precision(tc_precision)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            lib.ssb_vocoder_free(h)
            self._h = None

    def set_tensor_cores(self, enable=True):
        return bool(lib.ssb_vocoder_set_tensor_cores(self._h, 1 if enable else 0))

    def set_precision(self, mode: str):
        """Precision of the generator's tensor-core GEMMs (the ups and ResBlock convs on tensor cores, every layout):
        'split' (the default) or 'fp16' (single pass), as AcousticModel.set_mel_precision.  The output denoiser and the FFMA
        convs are unchanged."""
        if mode not in TC_PRECISIONS:
            raise ValueError(f"vocoder precision must be one of {sorted(TC_PRECISIONS)}, got {mode!r}")
        check(lib.ssb_vocoder_set_precision(self._h, TC_PRECISIONS[mode]), "ssb_vocoder_set_precision")
        self.precision = mode

    max_frames_per_call = 24000  # ~0.9 MB of stage buffers per frame: bounds the workspace to ~20 GB

    def generate(self, mel, f0, frame_offsets, rand_ini=None, src_noise=None, seed=0, denoise_c=None, seeds=None):
        """mel [sumF,80], f0 [sumF] or None (device, tight) -> wav [sumF*hop] (device).
        Large batches are processed in groups of utterances (results are per-utterance, so grouping is exact).
        denoise_c: the denoiser strength for this call (None = the vocoder's own ``denoise_c``); > 0 denoises every group
        in place right after it is generated.
        seeds: one seed per utterance (see utt_seeds) instead of `seed`: utterance b's wav is that of a B = 1 call with
        seed=seeds[b], however the batch is grouped.  rand_ini / src_noise cannot be combined with it."""
        fo = np.ascontiguousarray(frame_offsets, np.int32)
        B = len(fo) - 1
        c = self.denoise_c if denoise_c is None else float(denoise_c)
        keys = None
        if seeds is not None:
            keys = utt_seeds(seeds, B)
            if rand_ini is not None or src_noise is not None:
                raise ValueError("seeds: per-utterance seeds key the in-kernel noise; rand_ini / src_noise must be None")
        if B > 1 and int(fo[-1]) > self.max_frames_per_call:
            wav = torch.empty(int(fo[-1]) * self.hop, dtype=torch.float32, device=self.device)
            b0 = 0
            while b0 < B:
                b1 = b0 + 1
                while b1 < B and int(fo[b1 + 1] - fo[b0]) <= self.max_frames_per_call:
                    b1 += 1
                sub_fo = (fo[b0:b1 + 1] - fo[b0]).astype(np.int32)
                a, e = int(fo[b0]), int(fo[b1])
                w = self.generate(mel[a:e], None if f0 is None else f0[a:e], sub_fo,
                                  None if rand_ini is None else rand_ini[b0:b1].contiguous(),
                                  None if src_noise is None else src_noise[a * self.hop:e * self.hop], seed + b0, c,
                                  None if keys is None else keys[b0:b1])
                wav[a * self.hop:e * self.hop] = w
                b0 = b1
            return wav
        n = lib.ssb_vocoder_workspace_bytes(self._h, fo.ctypes.data, B)
        if n == 0:
            check(-1, "ssb_vocoder_workspace_bytes")
        ws = self._ws.get(n)
        wav = torch.empty(int(fo[-1]) * self.hop, dtype=torch.float32, device=self.device)
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        if keys is None:
            check(lib.ssb_hifigan_generate(self._h, _ptr(mel), _ptr(f0), fo.ctypes.data, B, _ptr(rand_ini),
                                           _ptr(src_noise), int(seed), _ptr(wav), _ptr(ws), ws.numel(), stream),
                  "ssb_hifigan_generate")
        else:
            check(lib.ssb_hifigan_generate_keyed(self._h, _ptr(mel), _ptr(f0), fo.ctypes.data, B, keys.ctypes.data,
                                                 _ptr(wav), _ptr(ws), ws.numel(), stream), "ssb_hifigan_generate_keyed")
        if c > 0:  # hifigan_nsf.py:73-74: only a positive strength runs the denoiser
            if self._denoiser is None:
                self._denoiser = WavDenoiser(self._denoise_hp if self._denoise_hp is not None else self.cfg, self.device)
            self._denoiser(wav, fo * self.hop, c, out=wav, workspace=self._ws)
        return wav


class WavDenoiser:
    """Spectral-subtraction denoiser of the vocoder output (ssb_wav_denoise_t): denoise(wav, v) of the reference
    (tasks/tts/vocoder_infer/hifigan_nsf.py:14-22), every utterance on its own.  Geometry from hp's fft_size / hop_size /
    win_size (defaults 1024 / 256 / 1024, as MelSpectrogram)."""

    def __init__(self, hp=None, device=None):
        _require_cuda()
        h = dict(fft_size=1024, hop_size=256, win_size=1024)
        h.update({k: v for k, v in (hp or {}).items() if k in h})
        self.hp = h
        self.device = torch.device(device if device is not None else "cuda:0")
        torch.cuda.set_device(self.device)
        handle = C.c_void_p()
        check(lib.ssb_wav_denoise_create(C.byref(handle), h["fft_size"], h["hop_size"], h["win_size"]), "ssb_wav_denoise_create")
        self._h = handle
        self._ws = _Workspace(self.device)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            lib.ssb_wav_denoise_free(h)
            self._h = None

    def set_tensor_cores(self, mode=1):
        """GEMM path: 1 / True = tensor cores for batches of >= 8 row tiles, FFMA below (default); 0 / False = fp32 FFMA
        always; 2 = tensor cores at every size (tests, measurement).  Returns the mode in effect."""
        return int(lib.ssb_wav_denoise_set_tensor_cores(self._h, int(mode)))

    def workspace_bytes(self, sample_offsets):
        so = np.ascontiguousarray(sample_offsets, np.int32)
        return int(lib.ssb_wav_denoise_workspace_bytes(self._h, so.ctypes.data, len(so) - 1))

    def __call__(self, wav, sample_offsets, v, out=None, workspace=None):
        """wav: device fp32 [sum n_b] (utterances concatenated, every n_b a positive multiple of hop_size), sample_offsets:
        [B+1].  Returns the denoised waveform (``out``, which may be ``wav`` itself, or a new tensor)."""
        so = np.ascontiguousarray(sample_offsets, np.int32)
        n = lib.ssb_wav_denoise_workspace_bytes(self._h, so.ctypes.data, len(so) - 1)
        if n == 0:
            check(-1, "ssb_wav_denoise_workspace_bytes")
        ws = (workspace or self._ws).get(n)
        out = torch.empty_like(wav) if out is None else out
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        check(lib.ssb_wav_denoise_forward(self._h, _ptr(wav), so.ctypes.data, len(so) - 1, float(v), _ptr(out), _ptr(ws),
                                          ws.numel(), stream), "ssb_wav_denoise_forward")
        return out


# unit-test granularity ops -------------------------------------------------------------------------
class MelSpectrogram:
    """log10-mel front-end of the reference audio (ssb_melspec_t): librosa_wav2spec of the reference
    (utils/audios/__init__.py:36-84) with the hparams of egs/stylesinger.yaml by default."""

    def __init__(self, hp=None, device=None, eps=1e-6, pad_reflect=False, power=False, log=True):
        """pad_reflect / power / log=False select the defaults of librosa.feature.melspectrogram instead of those of
        librosa_wav2spec (ssb_melspec_create_ex; the emotion encoder's features, data_gen/tts/emotion/audio.py:43-55)."""
        _require_cuda()
        h = dict(audio_sample_rate=48000, fft_size=1024, hop_size=256, win_size=1024, audio_num_mel_bins=80, fmin=20, fmax=24000)
        h.update({k: v for k, v in (hp or {}).items() if k in h})
        self.hp = h
        self.device = torch.device(device if device is not None else "cuda:0")
        torch.cuda.set_device(self.device)
        handle = C.c_void_p()
        check(lib.ssb_melspec_create_ex(C.byref(handle), h["audio_sample_rate"], h["fft_size"], h["hop_size"], h["win_size"],
                                        h["audio_num_mel_bins"], float(h["fmin"]), float(h["fmax"]), float(eps),
                                        int(bool(pad_reflect)), int(bool(power)), int(bool(log))), "ssb_melspec_create_ex")
        self._h = handle
        self._ws = _Workspace(self.device)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            lib.ssb_melspec_free(h)
            self._h = None

    def num_frames(self, n_samples):
        return int(lib.ssb_melspec_num_frames(self._h, int(n_samples)))

    def __call__(self, wavs):
        """wavs: list of 1-D float32 arrays / tensors (or one).  Returns a list of device tensors [frames, n_mels]."""
        single = not isinstance(wavs, (list, tuple))
        wavs = [wavs] if single else list(wavs)
        ts = [torch.as_tensor(np.asarray(w, dtype=np.float32) if not isinstance(w, torch.Tensor) else w, dtype=torch.float32).reshape(-1)
              for w in wavs]
        offs = np.concatenate([[0], np.cumsum([t.numel() for t in ts])]).astype(np.int32)
        wav = torch.cat(ts).to(self.device).contiguous() if ts else torch.zeros(0, device=self.device)
        frames = [self.num_frames(t.numel()) for t in ts]
        out = torch.empty(sum(frames), self.hp["audio_num_mel_bins"], dtype=torch.float32, device=self.device)
        n = lib.ssb_melspec_workspace_bytes(self._h, offs.ctypes.data, len(ts))
        if n == 0:
            check(-1, "ssb_melspec_workspace_bytes")
        ws = self._ws.get(n)
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        check(lib.ssb_melspec_forward(self._h, _ptr(wav), offs.ctypes.data, len(ts), _ptr(out), _ptr(ws), ws.numel(), stream),
              "ssb_melspec_forward")
        mels = list(torch.split(out, frames))
        return mels[0] if single else mels


class LstmEncoder:
    """LSTM utterance encoder of the reference audio (ssb_lstm_encoder_t): the reference's EmotionEncoder
    (data_gen/tts/emotion/model.py:10-77).  ``state_dict``: the encoder's own keys (``lstm.weight_ih_l0`` ..., optional
    ``linear.weight`` / ``linear.bias``), torch tensors or numpy arrays."""

    def __init__(self, state_dict, device=None):
        _require_cuda()
        self.device = torch.device(device if device is not None else "cuda:0")
        torch.cuda.set_device(self.device)
        sd = {k: np.ascontiguousarray(v.detach().cpu().float().numpy() if isinstance(v, torch.Tensor) else np.asarray(v, np.float32))
              for k, v in state_dict.items() if k.startswith(("lstm.", "linear."))}
        L = 0
        while "lstm.weight_ih_l%d" % L in sd:
            L += 1
        if L == 0:
            raise KeyError("state_dict has no lstm.weight_ih_l0")
        self.layers, self.hidden = L, sd["lstm.weight_hh_l0"].shape[1]
        self.n_in = sd["lstm.weight_ih_l0"].shape[1]
        for l in range(L):
            for k, shape in (("weight_ih", (4 * self.hidden, self.n_in if l == 0 else self.hidden)), ("weight_hh", (4 * self.hidden, self.hidden)),
                             ("bias_ih", (4 * self.hidden,)), ("bias_hh", (4 * self.hidden,))):
                name = "lstm.%s_l%d" % (k, l)
                if name not in sd or sd[name].shape != shape:
                    raise ValueError(f"{name}: expected shape {shape}, got {sd[name].shape if name in sd else None}")
        table = lambda k: (C.c_void_p * L)(*[sd["lstm.%s_l%d" % (k, l)].ctypes.data for l in range(L)])
        lw, lb = sd.get("linear.weight"), sd.get("linear.bias")
        self.embed = 0 if lw is None else lw.shape[0]
        if lw is not None and (lb is None or lw.shape != (self.embed, self.hidden) or lb.shape != (self.embed,)):
            raise ValueError("linear.weight / linear.bias shapes do not match the LSTM")
        handle = C.c_void_p()
        check(lib.ssb_lstm_encoder_create(C.byref(handle), self.n_in, self.hidden, L, table("weight_ih"), table("weight_hh"),
                                          table("bias_ih"), table("bias_hh"), self.embed,
                                          None if lw is None else lw.ctypes.data, None if lw is None else lb.ctypes.data),
              "ssb_lstm_encoder_create")
        self._h = handle
        self._ws = _Workspace(self.device)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            lib.ssb_lstm_encoder_free(h)
            self._h = None

    def __call__(self, frames, utt_offsets=None, want_embeds=False):
        """frames: [P, T, n_in] (device or host).  Returns a dict of device tensors: ``hidden`` [P, H] (EmotionEncoder.inference),
        ``embeds`` [P, E] (EmotionEncoder.forward, if want_embeds) and ``utt_embed`` [U, H] (normalised mean of ``hidden`` over
        partials utt_offsets[u] .. utt_offsets[u+1], if utt_offsets is given)."""
        x = torch.as_tensor(frames, dtype=torch.float32).to(self.device).contiguous()
        if x.dim() != 3 or x.shape[2] != self.n_in:
            raise ValueError(f"frames must be [partials, frames, {self.n_in}]")
        Pn, T = int(x.shape[0]), int(x.shape[1])
        out = {"hidden": torch.empty(Pn, self.hidden, dtype=torch.float32, device=self.device)}
        if want_embeds:
            if self.embed == 0:
                raise _lib.SsbError("encoder was created without the linear head (linear.weight / linear.bias)")
            out["embeds"] = torch.empty(Pn, self.embed, dtype=torch.float32, device=self.device)
        offs, U = None, 0
        if utt_offsets is not None:
            offs = np.ascontiguousarray(utt_offsets, np.int32)
            U = len(offs) - 1
            out["utt_embed"] = torch.empty(U, self.hidden, dtype=torch.float32, device=self.device)
        n = lib.ssb_lstm_encoder_workspace_bytes(self._h, Pn, T, U)
        if n == 0:
            check(-1, "ssb_lstm_encoder_workspace_bytes")
        ws = self._ws.get(n)
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        check(lib.ssb_lstm_encoder_forward(self._h, _ptr(x), Pn, T, None if offs is None else offs.ctypes.data, U, _ptr(out["hidden"]),
                                           _ptr(out.get("embeds")), _ptr(out.get("utt_embed")), _ptr(ws), ws.numel(), stream),
              "ssb_lstm_encoder_forward")
        return out


def _guarded(offsets, device):
    """Where the tight rows of the utterances at host offsets [B + 1] sit in the guard-banded layout of op_gemm and
    op_attention_ex: (row of each tight row, on `device`; the layout's row count).  Utterance b starts at row
    rs_b = 16 + off[b] + 16 b, and the layout has off[B] + 16 (B + 1) + 256 rows: 16 guard rows before and after every
    utterance, then 256 rows of tail slack (Seq::build, GUARD and TAIL_SLACK in csrc/common.cuh)."""
    off = np.ascontiguousarray(offsets, np.int64)
    B = len(off) - 1
    idx = np.arange(off[-1]) + 16 * np.repeat(np.arange(1, B + 1), np.diff(off))
    return torch.from_numpy(idx).to(device), int(off[-1]) + 16 * (B + 1) + 256


def _scatter(t, idx, rows):
    """Tight rows t in a zeroed fp32 [rows, ...] buffer at the rows idx of _guarded."""
    g = torch.zeros((rows,) + tuple(t.shape[1:]), dtype=torch.float32, device=idx.device)
    g[idx] = t.to(g)
    return g


def _planes(x):
    """fp16 hi / lo planes of fp32 x, bit for bit what k_split_planes writes: hi = fp16(x), lo = fp16(x - hi)."""
    hi = x.half()
    return hi, (x - hi.float()).half()


def op_conv1d(x, offsets, w, b, dilation=1, act=0):
    """One Conv1d on the fp32 FFMA GEMM (op_gemm path 0) over the tight rows x [sum L, Cin] of the utterances at host
    offsets [B + 1], with torch-layout weights w [N, Cin, k] and bias b [N] (or None).  act: 0 none, 1 relu, 2 gelu,
    3 leaky relu (slope 0.1), 4 tanh.  Returns the tight rows [sum L, N]."""
    idx, rows = _guarded(offsets, x.device)
    out = torch.empty(rows, w.shape[0], device=x.device)
    op_gemm(0, offsets, rows, w, b, dilation=dilation, a=_scatter(x, idx, rows), lda=x.shape[1], act=act, out=out,
            ldo=w.shape[0])
    return out[idx]


def op_conv1d_tc(x, offsets, w, b, dilation=1):
    """op_conv1d (without activation) on the tensor-core GEMM (op_gemm path 1, Cin % 64 == 0, N % 64 == 0), x split
    into fp16 hi / lo planes first."""
    idx, rows = _guarded(offsets, x.device)
    hi, lo = _planes(_scatter(x, idx, rows))
    out = torch.empty(rows, w.shape[0], device=x.device)
    op_gemm(1, offsets, rows, w, b, dilation=dilation, a_hi=hi, a_lo=lo, out=out, ldo=w.shape[0])
    return out[idx]


def _op_call(args, fields, fn, what):
    """Sets the keyword fields of a ctypes args struct (tensors by device pointer, a view's offset included; nothing is
    copied) and calls fn on it on the current stream of the tensors' device."""
    dev = None
    for name, v in fields.items():
        if isinstance(v, torch.Tensor):
            dev = v.device
            v = _ptr(v).value
        setattr(args, name, v)
    check(fn(C.byref(args), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), what)


def op_gemm(path, offsets, rows, w, b=None, dilation=1, gate=False, single_pass=False, **epi):
    """Exactly one conv_gemm (path 0, fp32 FFMA) or conv_gemm_tc (path 1, tensor cores) call (ssb_op_gemm) over
    caller-owned device tensors in the guard-banded layout of `offsets` with `rows` rows (utterance b at rows
    [rs_b, rs_b + L_b), rs_0 = 16, rs_{b+1} = rs_b + L_b + 16, plus 256 rows of tail slack).  w [N, Cin, k] / b [N]
    are torch-layout weights (gate=True: the DiffNet gate interleave).  epi: the A operand (a / lda / a_act / a_slope /
    a_scale on path 0, a_hi / a_lo on path 1) and the fields of ssb_op_gemm_args' epilogue; tensors are passed by
    pointer, nothing is copied.  single_pass=True (path 1 only): one hi*hi MMA per K step, the kernel of the 'fp16'
    tc_precision (a_lo is not read).  Returns nothing: the kernel writes into the given buffers."""
    _require_cuda()
    off = np.ascontiguousarray(offsets, np.int32)
    N, Cin, k = w.shape
    wc = w.detach().cpu().float().contiguous()
    bc = None if b is None else b.detach().cpu().float().contiguous()
    a = _lib.OpGemmArgs(path=path, frame_offsets=off.ctypes.data, B=len(off) - 1, rows=rows, Cin=Cin, N=N, k=k,
                        dilation=dilation, gate=int(gate), w_host=wc.data_ptr(), b_host=None if bc is None else bc.data_ptr(),
                        a_slope=0.1, a_scale=1.0, alpha=1.0, act_slope=0.1, beta=1.0, gamma=1.0, plane_slope=0.1,
                        single_pass=int(bool(single_pass)))
    _op_call(a, epi, lib.ssb_op_gemm, "ssb_op_gemm")


def op_attention_ex(path, q_offsets, k_offsets, rows_q, rows_k, scale, heads=2, **bufs):
    """Exactly one attention_kernel (path 0, fp32) or attention_tc_kernel (path 1, wgmma) call (ssb_op_attention_ex) over
    caller-owned device tensors in the guard-banded layouts of q_offsets (rows_q rows) and k_offsets (rows_k rows), the
    layout of op_gemm.  bufs: the operands (q / k / v on path 0, q_hi ... v_lo on path 1), keymask, out / oh / ol, and the
    ints ldq, qcol0, ldk, kcol0, ldv, vcol0, ldo, ldh; tensors are passed by pointer (a view's offset included), nothing
    is copied.  Returns nothing: the kernel writes into the given buffers."""
    _require_cuda()
    qo = np.ascontiguousarray(q_offsets, np.int32)
    ko = np.ascontiguousarray(k_offsets, np.int32)
    a = _lib.OpAttentionArgs(path=path, q_offsets=qo.ctypes.data, k_offsets=ko.ctypes.data, B=len(qo) - 1, rows_q=rows_q,
                             rows_k=rows_k, heads=heads, scale=float(scale))
    _op_call(a, bufs, lib.ssb_op_attention_ex, "ssb_op_attention_ex")


def op_attention(q, k, v, q_offsets, k_offsets, scale, tc=False, keymask=None):
    """Multi-head attention, 2 heads x 128, over tight rows: q [sum L, 256] of the query utterances at host q_offsets
    [B + 1], k / v [sum S, 256] of the key utterances at k_offsets; query utterance b attends to key utterance b.  On the
    fp32 kernel (op_attention_ex path 0), or with tc=True on the wgmma / TMA kernel (path 1, on fp16 hi / lo planes of q,
    k and v).  keymask: optional [sum S] tensor, 0 = masked key; an utterance whose keys are all masked (or that has no
    keys) gets NaN rows, as torch's softmax over all -inf does.  Returns the tight rows [sum L, 256]."""
    iq, rows_q = _guarded(q_offsets, q.device)
    ik, rows_k = _guarded(k_offsets, q.device)
    bufs = {}
    if keymask is not None:
        if keymask.shape != (k.shape[0],):
            raise ValueError(f"keymask must have shape ({k.shape[0]},), got {tuple(keymask.shape)}")
        bufs["keymask"] = _scatter(keymask, ik, rows_k)
    for name, t, idx, rows in (("q", q, iq, rows_q), ("k", k, ik, rows_k), ("v", v, ik, rows_k)):
        if tc:
            bufs[name + "_hi"], bufs[name + "_lo"] = _planes(_scatter(t, idx, rows))
        else:
            bufs[name] = _scatter(t, idx, rows)
    out = torch.empty(rows_q, 256, device=q.device)
    op_attention_ex(int(tc), q_offsets, k_offsets, rows_q, rows_k, scale, ldq=256, ldk=256, ldv=256, out=out, ldo=256,
                    **bufs)
    return out[iq]
