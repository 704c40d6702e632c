"""ctypes binding of libstylesinger_b200.so (include/stylesinger_b200.h).

There is deliberately NO fallback: if the CUDA library is missing or fails to load, importing this
module raises, and every compute entry point of the package is unavailable.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SSB_LIB_PATH: another build of the same library (A/B runs of two code states on one GPU box; must export the same symbols)
LIB_PATH = os.environ.get("SSB_LIB_PATH") or os.path.join(_HERE, "libstylesinger_b200.so")


class SsbError(RuntimeError):
    pass


class TensorDesc(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("ndim", C.c_int32), ("shape", C.c_int64 * 4)]


class HParams(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "hidden_size", "enc_layers", "dec_layers", "enc_ffn_kernel", "dec_ffn_kernel", "dur_layers", "dur_kernel",
        "n_tokens", "n_rq", "rq_depth", "mel_channels", "mel_layers", "mel_cycle", "f0_channels", "f0_layers",
        "f0_cycle", "mel_bins")]


class ModelSwitches(C.Structure):  # ssb_model_switches: hparams emo / style / umln / use_txt_cond, each 0 or 1
    _fields_ = [("emo", C.c_int32), ("style", C.c_int32), ("umln", C.c_int32), ("use_txt_cond", C.c_int32)]


class VocoderConfig(C.Structure):
    _fields_ = [("n_up", C.c_int32), ("up_rates", C.c_int32 * 8), ("up_kernels", C.c_int32 * 8),
                ("initial_channel", C.c_int32), ("n_res", C.c_int32), ("res_kernels", C.c_int32 * 4),
                ("res_dilations", (C.c_int32 * 3) * 4), ("use_pitch_embed", C.c_int32), ("sample_rate", C.c_int32)]


class VocoderConfigEx(C.Structure):
    """ssb_vocoder_config_ex: the VocoderConfig fields plus the ResBlock type (1 or 2)."""
    _fields_ = VocoderConfig._fields_ + [("resblock", C.c_int32)]


class AcousticInputs(C.Structure):
    _fields_ = [("B", C.c_int32),
                ("ph_offsets", C.c_void_p), ("frame_offsets", C.c_void_p), ("ref_offsets", C.c_void_p),
                ("txt_tokens", C.c_void_p), ("note", C.c_void_p), ("note_type", C.c_void_p), ("note_dur", C.c_void_p),
                ("spk_embed", C.c_void_p), ("emo_embed", C.c_void_p), ("ref_mels", C.c_void_p), ("ref_f0", C.c_void_p),
                ("mel2ph", C.c_void_p), ("dur", C.c_void_p), ("f0", C.c_void_p), ("uv", C.c_void_p),
                ("f0_gauss_noise", C.c_void_p * 2), ("f0_unif_noise", C.c_void_p * 2), ("mel_noise", C.c_void_p),
                ("seed", C.c_uint64), ("skip_mel_diffusion", C.c_int32), ("pndm_speedup", C.c_int32),
                ("spk_ids", C.c_void_p)]


class AcousticOutputs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "mel_out", "f0_denorm", "encoder_out", "style", "rq_codes", "pitch_pred", "decoder_inp", "coarse_mel",
        "diff_cond", "mel2ph", "spk_proj", "emo_proj")]


class OpGemmArgs(C.Structure):
    """ssb_op_gemm_args: one conv_gemm (path 0) or conv_gemm_tc (path 1) call over caller-owned device buffers."""
    _fields_ = [("path", C.c_int32), ("frame_offsets", C.c_void_p), ("B", C.c_int32), ("rows", C.c_int64),
                ("Cin", C.c_int32), ("N", C.c_int32), ("k", C.c_int32), ("dilation", C.c_int32), ("gate", C.c_int32),
                ("w_host", C.c_void_p), ("b_host", C.c_void_p),
                ("a", C.c_void_p), ("lda", C.c_int32), ("a_act", C.c_int32), ("a_slope", C.c_float), ("a_scale", C.c_float),
                ("a_hi", C.c_void_p), ("a_lo", C.c_void_p),
                ("mode", C.c_int32), ("add", C.c_void_p), ("ld_add", C.c_int32), ("alpha", C.c_float), ("act", C.c_int32),
                ("act_slope", C.c_float), ("res", C.c_void_p), ("ld_res", C.c_int32), ("beta", C.c_float),
                ("rowmask", C.c_void_p), ("out", C.c_void_p), ("ldo", C.c_int32), ("accum", C.c_int32), ("gamma", C.c_float),
                ("out2", C.c_void_p), ("ldo2", C.c_int32), ("vec1", C.c_void_p), ("vec2", C.c_void_p),
                ("oh", C.c_void_p), ("ol", C.c_void_p), ("ldh", C.c_int32), ("plane_act", C.c_int32),
                ("plane_slope", C.c_float), ("skip", C.c_void_p), ("ld_skip", C.c_int32), ("C", C.c_int32),
                ("skip_init", C.c_int32), ("rh", C.c_void_p), ("rl", C.c_void_p), ("ld_rh", C.c_int32),
                ("skip_tiled", C.c_int32), ("out_nb", C.c_int32), ("out_bs", C.c_int64), ("sh", C.c_void_p),
                ("sl", C.c_void_p), ("n_valid", C.c_int32), ("single_pass", C.c_int32)]


class OpAttentionArgs(C.Structure):
    """ssb_op_attention_args: one attention_kernel (path 0) or attention_tc_kernel (path 1) call over caller-owned
    device buffers."""
    _fields_ = [("path", C.c_int32), ("q_offsets", C.c_void_p), ("k_offsets", C.c_void_p), ("B", C.c_int32),
                ("rows_q", C.c_int64), ("rows_k", C.c_int64), ("heads", C.c_int32), ("scale", C.c_float),
                ("keymask", C.c_void_p), ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p),
                ("q_hi", C.c_void_p), ("q_lo", C.c_void_p), ("k_hi", C.c_void_p), ("k_lo", C.c_void_p),
                ("v_hi", C.c_void_p), ("v_lo", C.c_void_p),
                ("ldq", C.c_int32), ("qcol0", C.c_int32), ("ldk", C.c_int32), ("kcol0", C.c_int32), ("ldv", C.c_int32),
                ("vcol0", C.c_int32), ("out", C.c_void_p), ("ldo", C.c_int32), ("oh", C.c_void_p), ("ol", C.c_void_p),
                ("ldh", C.c_int32)]


# every symbol declared in include/stylesinger_b200.h (tests/test_abi.py checks this list against the header)
EXPORTS = [
    "ssb_version", "ssb_last_error", "ssb_model_create", "ssb_model_free", "ssb_model_set_schedule",
    "ssb_durations_workspace_bytes", "ssb_predict_durations", "ssb_acoustic_workspace_bytes", "ssb_acoustic_forward",
    "ssb_mel_diffusion_workspace_bytes", "ssb_mel_diffusion_sample", "ssb_denoiser_eval", "ssb_f0_diffusion_sample",
    "ssb_rvq_lookup", "ssb_vocoder_create", "ssb_vocoder_free", "ssb_vocoder_workspace_bytes", "ssb_hifigan_generate",
    "ssb_mel_postprocess", "ssb_launch_count",
    "ssb_model_set_tensor_cores", "ssb_model_set_persistent", "ssb_model_set_fft_tensor_cores",
    "ssb_vocoder_set_tensor_cores", "ssb_variant_launch_count", "ssb_variant_names", "ssb_tensor_map_cache_stats",
    "ssb_model_set_persistent_groups", "ssb_mel_diffusion_plms_workspace_bytes",
    "ssb_mel_diffusion_sample_plms", "ssb_fft_workspace_bytes", "ssb_fft_encoder", "ssb_fft_decoder",
    "ssb_get_style_workspace_bytes", "ssb_get_style", "ssb_set_attention_tensor_cores",
    "ssb_melspec_create", "ssb_melspec_free", "ssb_melspec_num_frames", "ssb_melspec_workspace_bytes", "ssb_melspec_forward",
    "ssb_melspec_create_ex", "ssb_lstm_encoder_create", "ssb_lstm_encoder_free", "ssb_lstm_encoder_workspace_bytes", "ssb_lstm_encoder_forward",
    "ssb_model_create_ex", "ssb_mel_prodiff_workspace_bytes", "ssb_mel_prodiff_sample",
    "ssb_model_create_ex2", "ssb_pitch_predictor_workspace_bytes", "ssb_pitch_predictor",
    "ssb_wav_denoise_create", "ssb_wav_denoise_free", "ssb_wav_denoise_workspace_bytes", "ssb_wav_denoise_forward",
    "ssb_wav_denoise_set_tensor_cores",
    "ssb_model_set_mel_k_step",
    "ssb_acoustic_forward_keyed", "ssb_hifigan_generate_keyed",
    "ssb_vocoder_create_ex",
    "ssb_op_gemm",
    "ssb_op_attention_ex", "ssb_attention_launch_count",
    "ssb_model_create_ex3",
    "ssb_model_set_mel_precision", "ssb_vocoder_set_precision",
    "ssb_model_create_ex4",
]


def _load():
    if not os.path.exists(LIB_PATH):
        raise SsbError(f"{LIB_PATH} not found: build it with `python -m stylesinger_b200.build` "
                       f"(nvcc, sm_90a). There is no CPU / PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, i32, u64, sz = C.c_void_p, C.c_int32, C.c_uint64, C.c_size_t
    P = C.POINTER
    sig = {
        "ssb_version": (C.c_int, []),
        "ssb_last_error": (C.c_char_p, []),
        "ssb_model_create": (C.c_int, [P(vp), P(TensorDesc), i32, P(HParams)]),
        "ssb_model_create_ex": (C.c_int, [P(vp), P(TensorDesc), i32, P(HParams), i32]),
        "ssb_model_create_ex2": (C.c_int, [P(vp), P(TensorDesc), i32, P(HParams), i32, i32]),
        "ssb_model_create_ex3": (C.c_int, [P(vp), P(TensorDesc), i32, P(HParams), i32, i32, P(ModelSwitches)]),
        "ssb_model_create_ex4": (C.c_int, [P(vp), P(TensorDesc), i32, P(HParams), i32, i32, P(ModelSwitches), i32]),
        "ssb_pitch_predictor_workspace_bytes": (sz, [vp, vp, i32]),
        "ssb_pitch_predictor": (C.c_int, [vp, i32, vp, vp, i32, vp, vp, sz, vp]),
        "ssb_model_free": (None, [vp]),
        "ssb_model_set_schedule": (C.c_int, [vp, i32, i32, vp, vp, vp, vp]),
        "ssb_model_set_mel_k_step": (C.c_int, [vp, i32]),
        "ssb_durations_workspace_bytes": (sz, [vp, P(AcousticInputs)]),
        "ssb_predict_durations": (C.c_int, [vp, P(AcousticInputs), vp, vp, vp, sz, vp]),
        "ssb_acoustic_workspace_bytes": (sz, [vp, P(AcousticInputs)]),
        "ssb_acoustic_forward": (C.c_int, [vp, P(AcousticInputs), P(AcousticOutputs), vp, sz, vp]),
        "ssb_acoustic_forward_keyed": (C.c_int, [vp, P(AcousticInputs), vp, P(AcousticOutputs), vp, sz, vp]),
        "ssb_mel_diffusion_workspace_bytes": (sz, [vp, vp, i32]),
        "ssb_mel_diffusion_sample": (C.c_int, [vp, vp, vp, vp, i32, vp, u64, vp, vp, sz, vp]),
        "ssb_mel_prodiff_workspace_bytes": (sz, [vp, vp, i32]),
        "ssb_mel_prodiff_sample": (C.c_int, [vp, vp, vp, i32, vp, u64, vp, vp, sz, vp]),
        "ssb_mel_diffusion_plms_workspace_bytes": (sz, [vp, vp, i32]),
        "ssb_mel_diffusion_sample_plms": (C.c_int, [vp, vp, vp, vp, i32, vp, u64, i32, vp, vp, sz, vp]),
        "ssb_denoiser_eval": (C.c_int, [vp, i32, vp, vp, i32, vp, vp, i32, vp, vp, sz, vp]),
        "ssb_f0_diffusion_sample": (C.c_int, [vp, i32, vp, vp, vp, vp, i32, vp, vp, u64, vp, vp, vp, sz, vp]),
        "ssb_rvq_lookup": (C.c_int, [vp, vp, vp, i32, vp, vp, vp, sz, vp]),
        "ssb_vocoder_create": (C.c_int, [P(vp), P(TensorDesc), i32, P(VocoderConfig)]),
        "ssb_vocoder_create_ex": (C.c_int, [P(vp), P(TensorDesc), i32, P(VocoderConfigEx)]),
        "ssb_vocoder_free": (None, [vp]),
        "ssb_vocoder_workspace_bytes": (sz, [vp, vp, i32]),
        "ssb_hifigan_generate": (C.c_int, [vp, vp, vp, vp, i32, vp, vp, u64, vp, vp, sz, vp]),
        "ssb_hifigan_generate_keyed": (C.c_int, [vp, vp, vp, vp, i32, vp, vp, vp, sz, vp]),
        "ssb_mel_postprocess": (C.c_int, [vp, C.c_int64, C.c_float, C.c_float, vp, vp]),
        "ssb_launch_count": (C.c_int64, []),
        "ssb_model_set_tensor_cores": (C.c_int, [vp, i32]),
        "ssb_model_set_persistent": (C.c_int, [vp, i32]),
        "ssb_model_set_persistent_groups": (C.c_int, [vp, i32]),
        "ssb_model_set_fft_tensor_cores": (C.c_int, [vp, i32]),
        "ssb_vocoder_set_tensor_cores": (C.c_int, [vp, i32]),
        "ssb_model_set_mel_precision": (C.c_int, [vp, i32]),
        "ssb_vocoder_set_precision": (C.c_int, [vp, i32]),
        "ssb_op_gemm": (C.c_int, [P(OpGemmArgs), vp]),
        "ssb_op_attention_ex": (C.c_int, [P(OpAttentionArgs), vp]),
        "ssb_attention_launch_count": (C.c_int64, [i32]),
        "ssb_fft_workspace_bytes": (sz, [vp, i32, vp, i32]),
        "ssb_fft_encoder": (C.c_int, [vp, vp, vp, i32, vp, vp, sz, vp]),
        "ssb_fft_decoder": (C.c_int, [vp, vp, vp, i32, vp, vp, sz, vp]),
        "ssb_get_style_workspace_bytes": (sz, [vp, vp, vp, i32]),
        "ssb_get_style": (C.c_int, [vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, sz, vp]),
        "ssb_variant_launch_count": (C.c_int64, [C.c_char_p]),
        "ssb_variant_names": (i32, [C.c_char_p, i32]),
        "ssb_tensor_map_cache_stats": (None, [P(C.c_int64), P(C.c_int64)]),
        "ssb_set_attention_tensor_cores": (i32, [i32]),
        "ssb_melspec_create": (C.c_int, [P(vp), i32, i32, i32, i32, i32, C.c_float, C.c_float, C.c_float]),
        "ssb_melspec_create_ex": (C.c_int, [P(vp), i32, i32, i32, i32, i32, C.c_float, C.c_float, C.c_float, i32, i32, i32]),
        "ssb_melspec_free": (None, [vp]),
        "ssb_melspec_num_frames": (i32, [vp, C.c_int64]),
        "ssb_melspec_workspace_bytes": (sz, [vp, vp, i32]),
        "ssb_melspec_forward": (C.c_int, [vp, vp, vp, i32, vp, vp, sz, vp]),
        "ssb_lstm_encoder_create": (C.c_int, [P(vp), i32, i32, i32, vp, vp, vp, vp, i32, vp, vp]),
        "ssb_lstm_encoder_free": (None, [vp]),
        "ssb_lstm_encoder_workspace_bytes": (sz, [vp, i32, i32, i32]),
        "ssb_lstm_encoder_forward": (C.c_int, [vp, vp, i32, i32, vp, i32, vp, vp, vp, vp, sz, vp]),
        "ssb_wav_denoise_create": (C.c_int, [P(vp), i32, i32, i32]),
        "ssb_wav_denoise_free": (None, [vp]),
        "ssb_wav_denoise_workspace_bytes": (sz, [vp, vp, i32]),
        "ssb_wav_denoise_forward": (C.c_int, [vp, vp, vp, i32, C.c_float, vp, vp, sz, vp]),
        "ssb_wav_denoise_set_tensor_cores": (C.c_int, [vp, i32]),
    }
    for name in EXPORTS:
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype, fn.argtypes = sig[name]
    return lib


lib = _load()


def variant_launches():
    """{kernel variant name: launches so far} of the tensor-core GEMM dispatcher (ssb_variant_names / _launch_count)."""
    buf = C.create_string_buffer(4096)
    lib.ssb_variant_names(buf, 4096)
    names = [n for n in buf.value.decode().split(";") if n]
    return {n: int(lib.ssb_variant_launch_count(n.encode())) for n in names}


def check(rc, what=""):
    if rc != 0:
        msg = lib.ssb_last_error()
        raise SsbError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")
