"""Synthetic checkpoints and synthetic inputs (no network: there are no released weights here).

* ``acoustic_state_dict`` / ``vocoder_state_dict`` build state dicts with EXACTLY the parameter
  and buffer names/shapes of the reference modules (``StyleSinger`` —
  reference modules/StyleSinger/stylesinger.py:46-117 — and ``HifiGanGenerator`` —
  reference modules/hifigan/hifigan_nsf.py:104-142, weight-norm ``weight_g/weight_v`` form), so that
  (a) released checkpoints and these synthetic ones go through the same loader, and
  (b) tools/make_golden.py can ``load_state_dict(strict=True)`` them into the reference.
  The init is deliberately NOT the reference's: freshly constructed reference weights are
  degenerate for parity testing (zero-initialised denoiser output projections, N(0,0.01) vocoder
  convs, SURVEY.md §0.5), so every tensor is fan-in scaled to give O(1) activations.
* ``make_utterance`` / ``make_batch`` generate the seeded synthetic inputs of SURVEY.md §8(d).

Everything here is deterministic given the seed (torch CPU generator).
"""
import math
from collections import OrderedDict

import numpy as np
import torch

from .hparams import DEFAULT_VOCODER_CONFIG, resolve
from .schedules import gaussian_schedule, multinomial_schedule, prodiff_schedule

N_TOKENS = 61  # 58 phones + <pad>,<EOS>,<UNK> (reference ZH_checkpoint_phone_set.json)


# ----------------------------------------------------------------------------------------------
# parameter shape tables
# ----------------------------------------------------------------------------------------------
def _enc_sa_layer(p, H, k):
    return [(p + "layer_norm1.weight", (H,)), (p + "layer_norm1.bias", (H,)),
            (p + "self_attn.in_proj_weight", (3 * H, H)), (p + "self_attn.out_proj.weight", (H, H)),
            (p + "layer_norm2.weight", (H,)), (p + "layer_norm2.bias", (H,)),
            (p + "ffn.ffn_1.weight", (4 * H, H, k)), (p + "ffn.ffn_1.bias", (4 * H,)),
            (p + "ffn.ffn_2.weight", (H, 4 * H)), (p + "ffn.ffn_2.bias", (H,))]


def _predictor(p, H, n_layers, k, odim):
    out = []
    for i in range(n_layers):
        out += [(f"{p}conv.{i}.1.weight", (H, H, k)), (f"{p}conv.{i}.1.bias", (H,)),
                (f"{p}conv.{i}.3.weight", (H,)), (f"{p}conv.{i}.3.bias", (H,))]
    out += [(p + "linear.weight", (odim, H)), (p + "linear.bias", (odim,))]
    return out


def _diffnet(p, C, L, in_dims, out_dims, H, ddiff):
    out = []
    if ddiff:
        out += [(p + "input_projection.weight", (C // 2, in_dims, 1)), (p + "input_projection.bias", (C // 2,)),
                (p + "uv_embed.weight", (2, C // 2))]
    else:
        out += [(p + "input_projection.weight", (C, in_dims, 1)), (p + "input_projection.bias", (C,))]
    out += [(p + "mlp.0.weight", (4 * C, C)), (p + "mlp.0.bias", (4 * C,)),
            (p + "mlp.2.weight", (C, 4 * C)), (p + "mlp.2.bias", (C,))]
    for i in range(L):
        q = f"{p}residual_layers.{i}."
        out += [(q + "dilated_conv.weight", (2 * C, C, 3)), (q + "dilated_conv.bias", (2 * C,)),
                (q + "diffusion_projection.weight", (C, C)), (q + "diffusion_projection.bias", (C,)),
                (q + "conditioner_projection.weight", (2 * C, H, 1)), (q + "conditioner_projection.bias", (2 * C,)),
                (q + "output_projection.weight", (2 * C, C, 1)), (q + "output_projection.bias", (2 * C,))]
    out += [(p + "skip_projection.weight", (C, C, 1)), (p + "skip_projection.bias", (C,)),
            (p + "output_projection.weight", (out_dims, C, 1)), (p + "output_projection.bias", (out_dims,))]
    return out


_GAUSS_BUFS = ["betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod",
               "sqrt_one_minus_alphas_cumprod", "log_one_minus_alphas_cumprod", "sqrt_recip_alphas_cumprod",
               "sqrt_recipm1_alphas_cumprod", "posterior_variance", "posterior_log_variance_clipped",
               "posterior_mean_coef1", "posterior_mean_coef2"]
_MULTI_BUFS = ["log_alpha", "log_1_min_alpha", "log_cumprod_alpha", "log_1_min_cumprod_alpha"]


def acoustic_param_shapes(hp):
    """Ordered (name, shape) list in the reference's own state_dict order."""
    H = hp["hidden_size"]
    out = [("encoder_embed_tokens.weight", (N_TOKENS, H))]
    for i in range(hp["enc_layers"]):
        out += _enc_sa_layer(f"encoder.layers.{i}.op.", H, hp["enc_ffn_kernel_size"])
    out += [("encoder.layer_norm.weight", (H,)), ("encoder.layer_norm.bias", (H,)),
            ("encoder.embed_tokens.weight", (N_TOKENS, H)), ("encoder.embed_positions._float_tensor", (1,)),
            ("decoder.pos_embed_alpha", (1,)), ("decoder.embed_positions._float_tensor", (1,))]
    for i in range(hp["dec_layers"]):
        out += _enc_sa_layer(f"decoder.layers.{i}.op.", H, hp["dec_ffn_kernel_size"])
    out += [("decoder.layer_norm.weight", (H,)), ("decoder.layer_norm.bias", (H,)),
            ("mel_out.weight", (80, H)), ("mel_out.bias", (80,))]
    if hp["use_spk_id"]:  # Embedding(num_spk + 1, H) tables, no bias (fs2.py:37-41)
        rows = hp["num_spk"] + 1
        out += [("spk_embed_proj.weight", (rows, H))]
        if hp.get("use_split_spk_id"):
            out += [("spk_embed_f0.weight", (rows, H)), ("spk_embed_dur.weight", (rows, H))]
    else:
        out += [("spk_embed_proj.weight", (H, 256)), ("spk_embed_proj.bias", (H,))]
    out += _predictor("dur_predictor.", H, hp["dur_predictor_layers"], hp["dur_predictor_kernel"], 1)
    out += [("pitch_embed.weight", (300, H)), ("pitch_predictor.pos_embed_alpha", (1,))]
    # constructed by FastSpeech2 (unused with gmdiff); f0_gen 'conv' rebuilds it in place with the same shapes
    out += _predictor("pitch_predictor.", H, 5, hp["predictor_kernel"], 2)
    out += [("pitch_predictor.embed_positions._float_tensor", (1,)),
            ("note_encoder.emb.weight", (100, H)), ("note_encoder.type_emb.weight", (5, H)),
            ("note_encoder.dur_ln.weight", (H, 1)), ("note_encoder.dur_ln.bias", (H,))]
    if hp["emo"]:
        out += [("emo_embed_proj.weight", (H, hp["emo_size"])), ("emo_embed_proj.bias", (H,))]
    if hp["umln"]:
        out += [("norm.affine_layer.linear_layer.weight", (2 * H, H)), ("norm.affine_layer.linear_layer.bias", (2 * H,))]
    if hp["style"]:
        out += _style_modules(hp, H)
    Cf, Lf, Tf = hp["f0_residual_channels"], hp["f0_residual_layers"], hp["f0_timesteps"]
    if hp["f0_gen"] == "conv":  # StyleSinger.__init__ (stylesinger.py:73-82): a second PitchPredictor, no F0 diffusion
        out += [("pitch_inpainter_predictor.pos_embed_alpha", (1,))]
        out += _predictor("pitch_inpainter_predictor.", H, 5, hp["predictor_kernel"], 2)
        out += [("pitch_inpainter_predictor.embed_positions._float_tensor", (1,))]
    f0_nets = () if hp["f0_gen"] == "conv" else (("gm_diffnet", "f0_gen"), ("gm_diffnet_inpainte", "f0_gen_inpainte"))
    for net, gen in f0_nets:
        out += _diffnet(net + ".", Cf, Lf, 1, 3, H, True)
        out += [(f"{gen}.{b}", (Tf,)) for b in _MULTI_BUFS]
        out += [(f"{gen}.Lt_history", (Tf,)), (f"{gen}.Lt_count", (Tf,))]
        out += [(f"{gen}.{b}", (Tf,)) for b in _GAUSS_BUFS]
        out += _diffnet(gen + "._denoise_fn.", Cf, Lf, 1, 3, H, True)
    T = hp["timesteps"]
    if hp["decoder"] == "fft":  # stylesinger.py:92-117: neither ln_proj / postdiff nor diff_decoder
        return out + [("embed_positions._float_tensor", (1,))]
    if hp["decoder"] == "prodiff":  # ProDiffusion (stylesinger.py:111-117, prodiff.py:59-117): buffers of length T+1
        out += [("embed_positions._float_tensor", (1,)), ("diff_decoder.timesteps", ()), ("diff_decoder.timescale", ())]
        out += [(f"diff_decoder.{b}", (T + 1,)) for b in _GAUSS_BUFS]
        out += [("diff_decoder.spec_min", (1, 1, 80)), ("diff_decoder.spec_max", (1, 1, 80))]
        out += _diffnet("diff_decoder.denoise_fn.", hp["residual_channels"], hp["residual_layers"], 80, 80, H, False)
        return out
    cond_hs = 80 + H * (1 + hp["use_txt_cond"] + hp["emo"] + hp["style"])  # stylesinger.py:92-100
    out += [("embed_positions._float_tensor", (1,)), ("ln_proj.weight", (H, cond_hs)), ("ln_proj.bias", (H,))]
    out += [(f"postdiff.{b}", (T,)) for b in _GAUSS_BUFS]
    out += [("postdiff.spec_min", (1, 1, 80)), ("postdiff.spec_max", (1, 1, 80))]
    out += _diffnet("postdiff.denoise_fn.", hp["residual_channels"], hp["residual_layers"], 80, 80, H, False)
    return out


def _style_modules(hp, H):
    """LocalStyleAdaptor, l1 and ProsodyAligner (stylesinger.py:61-64): built only with hparams['style']."""
    out = []
    for i in range(5):
        for j in range(2):
            q = f"style_extractor.encoder.res_blocks.{i}.blocks.{j}."
            out += [(q + "0.weight", (80,)), (q + "0.bias", (80,)),
                    (q + "1.weight", (160, 80, 5)), (q + "1.bias", (160,)),
                    (q + "4.weight", (80, 160, 1)), (q + "4.bias", (80,))]
    out += [("style_extractor.encoder.last_norm.weight", (80,)), ("style_extractor.encoder.last_norm.bias", (80,)),
            ("style_extractor.encoder.post_net1.weight", (H, 80, 3)), ("style_extractor.encoder.post_net1.bias", (H,))]
    for d in range(hp["rq_depth"]):
        q = f"style_extractor.rqvae.codebooks.{d}."
        out += [(q + "weight", (hp["nRQ"] + 1, H)), (q + "cluster_size_ema", (hp["nRQ"],)),
                (q + "embed_ema", (hp["nRQ"], H))]
    for i in range(4):
        out += [(f"style_extractor.wavenet.in_layers.{i}.bias", (160,)),
                (f"style_extractor.wavenet.in_layers.{i}.weight_g", (160, 1, 1)),
                (f"style_extractor.wavenet.in_layers.{i}.weight_v", (160, 80, 3))]
    for i in range(4):
        c = 160 if i < 3 else 80
        out += [(f"style_extractor.wavenet.res_skip_layers.{i}.bias", (c,)),
                (f"style_extractor.wavenet.res_skip_layers.{i}.weight_g", (c, 1, 1)),
                (f"style_extractor.wavenet.res_skip_layers.{i}.weight_v", (c, 80, 1))]
    out += [("style_extractor.wavenet.cond_layer.bias", (640,)),
            ("style_extractor.wavenet.cond_layer.weight_g", (640, 1, 1)),
            ("style_extractor.wavenet.cond_layer.weight_v", (640, 80, 1)),
            ("l1.weight", (H, 2 * H)), ("l1.bias", (H,))]
    for i in range(2):
        q = f"align.layers.{i}."
        out += [(q + "multihead_attn.in_proj_weight", (3 * H, H)), (q + "multihead_attn.in_proj_bias", (3 * H,)),
                (q + "multihead_attn.out_proj.weight", (H, H)), (q + "multihead_attn.out_proj.bias", (H,)),
                (q + "linear1.weight", (2048, H)), (q + "linear1.bias", (2048,)),
                (q + "norm1.weight", (H,)), (q + "norm1.bias", (H,)),
                (q + "linear2.weight", (H, 2048)), (q + "linear2.bias", (H,)),
                (q + "norm2.weight", (H,)), (q + "norm2.bias", (H,))]
    return out


def vocoder_param_shapes(h):
    """HifiGanGenerator state_dict (weight-norm form), reference modules/hifigan/hifigan_nsf.py:104-142."""
    C0 = h["upsample_initial_channel"]
    out = []
    if h["use_pitch_embed"]:
        out += [("m_source.l_linear.weight", (1, 9)), ("m_source.l_linear.bias", (1,))]
        rates = h["upsample_rates"]
        for i in range(len(rates)):
            c = C0 // (2 ** (i + 1))
            if i + 1 < len(rates):
                s = int(np.prod(rates[i + 1:]))
                out += [(f"noise_convs.{i}.weight", (c, 1, 2 * s)), (f"noise_convs.{i}.bias", (c,))]
            else:
                out += [(f"noise_convs.{i}.weight", (c, 1, 1)), (f"noise_convs.{i}.bias", (c,))]
    out += [("conv_pre.bias", (C0,)), ("conv_pre.weight_g", (C0, 1, 1)), ("conv_pre.weight_v", (C0, 80, 7))]
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        c = C0 // (2 ** (i + 1))
        out += [(f"ups.{i}.bias", (c,)), (f"ups.{i}.weight_g", (2 * c, 1, 1)), (f"ups.{i}.weight_v", (2 * c, c, k))]
    nk = len(h["resblock_kernel_sizes"])
    # ResBlock1 (hifigan_nsf.py:30-66): convs1.{0,1,2} then convs2.{0,1,2}; ResBlock2 (:69-90, resblock != '1'): convs.{0,1}
    groups = (("convs1", 3), ("convs2", 3)) if str(h.get("resblock", "1")) == "1" else (("convs", 2),)
    for i in range(len(h["upsample_rates"])):
        c = C0 // (2 ** (i + 1))
        for j, k in enumerate(h["resblock_kernel_sizes"]):
            for grp, n_conv in groups:
                for m in range(n_conv):
                    q = f"resblocks.{i * nk + j}.{grp}.{m}."
                    out += [(q + "bias", (c,)), (q + "weight_g", (c, 1, 1)), (q + "weight_v", (c, c, k))]
    cl = C0 // (2 ** len(h["upsample_rates"]))
    out += [("conv_post.bias", (1,)), ("conv_post.weight_g", (1, 1, 1)), ("conv_post.weight_v", (1, cl, 7))]
    return out


# ----------------------------------------------------------------------------------------------
# initialisation
# ----------------------------------------------------------------------------------------------
def _is_norm_weight(name):
    tail = name.split(".")
    if name.endswith(".weight"):
        if any(s in name for s in ("layer_norm", "norm1.", "norm2.", "last_norm")):
            return True
        if "conv." in name and tail[-2] == "3":  # predictor LayerNorm (Sequential index 3)
            return True
        if "res_blocks" in name and tail[-2] == "0":  # ConvBlocks LayerNorm (Sequential index 0)
            return True
    return False


def _is_norm_bias(name):
    return name.endswith(".bias") and _is_norm_weight(name[:-5] + ".weight")


def acoustic_state_dict(hp=None, seed=0):
    hp = resolve(hp)
    g = torch.Generator().manual_seed(seed)
    H = hp["hidden_size"]
    sd = OrderedDict()
    shapes = acoustic_param_shapes(hp)
    sched = {"f0": (gaussian_schedule(hp["f0_timesteps"], hp["f0_max_beta"]),
                    multinomial_schedule(hp["f0_timesteps"], hp["f0_max_beta"])),
             "mel": (gaussian_schedule(hp["timesteps"], hp["max_beta"]), None)}
    if hp["decoder"] == "prodiff":
        sched["mel"] = (prodiff_schedule(hp["timesteps"], hp["schedule_type"]), None)
    for name, shape in shapes:
        base = name.split(".")[-1]
        if name.endswith("_float_tensor"):
            t = torch.zeros(1)
        elif name.endswith("pos_embed_alpha"):
            t = torch.ones(1)
        elif name == "diff_decoder.timesteps":
            t = torch.tensor(float(hp["timesteps"]))
        elif name == "diff_decoder.timescale":
            t = torch.tensor(float(hp.get("timescale", 1)))
        elif name.split(".")[0] in ("f0_gen", "f0_gen_inpainte", "postdiff", "diff_decoder") and base in _GAUSS_BUFS:
            s = sched["f0" if name.startswith("f0_gen") else "mel"][0]
            t = torch.from_numpy(s[base].copy())
        elif base in _MULTI_BUFS:
            t = torch.from_numpy(sched["f0"][1][base].copy())
        elif base in ("Lt_history", "Lt_count"):
            t = torch.zeros(shape)
        elif base == "spec_min":
            t = torch.tensor(hp["spec_min"], dtype=torch.float32)[None, None, :hp["keep_bins"]]
        elif base == "spec_max":
            t = torch.tensor(hp["spec_max"], dtype=torch.float32)[None, None, :hp["keep_bins"]]
        elif _is_norm_weight(name):
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif _is_norm_bias(name):
            t = 0.1 * torch.randn(shape, generator=g)
        elif name in ("encoder_embed_tokens.weight", "pitch_embed.weight", "note_encoder.emb.weight",
                      "note_encoder.type_emb.weight"):
            t = torch.randn(shape, generator=g) * H ** -0.5
            t[0] = 0  # padding_idx row
        elif name == "encoder.embed_tokens.weight":
            t = sd["encoder_embed_tokens.weight"]  # same Parameter in the reference
        elif "uv_embed" in name:
            t = torch.randn(shape, generator=g) * 0.5
        elif "rqvae.codebooks" in name and base == "weight":
            t = torch.randn(shape, generator=g) * 0.6
            t[-1] = 0  # padding_idx = n_embed
        elif base == "cluster_size_ema":
            t = torch.ones(shape)
        elif base == "embed_ema":
            t = sd[name[:-len("embed_ema")] + "weight"][:-1].clone()
        elif base == "weight_g":
            v_shape = dict(shapes)[name[:-1] + "v"]
            fan_in = int(np.prod(v_shape[1:]))
            # ||v|| per out channel ~ 1 for v ~ N(0, 1/fan_in); g jitters around it
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif base == "weight_v":
            fan_in = int(np.prod(shape[1:]))
            t = torch.randn(shape, generator=g) / math.sqrt(fan_in)
        elif name == "dur_predictor.linear.weight":
            t = torch.randn(shape, generator=g) * (0.05 / math.sqrt(H))
        elif name == "dur_predictor.linear.bias":
            t = torch.full(shape, math.log(1.0 + 8.0))
        elif name.endswith("output_projection.weight") and "residual_layers" not in name:
            t = torch.randn(shape, generator=g) / 16.0  # SURVEY §8(c) recipe (reference zero-inits this)
        elif base == "bias" or name.endswith("in_proj_bias"):
            t = 0.05 * torch.randn(shape, generator=g)
        else:  # dense / conv weights: fan-in scaled normal
            fan_in = int(np.prod(shape[1:])) if len(shape) > 1 else shape[0]
            t = torch.randn(shape, generator=g) / math.sqrt(fan_in)
        assert tuple(t.shape) == tuple(shape), (name, t.shape, shape)
        sd[name] = t.float().contiguous()
    # the reference registers each F0 denoiser twice (gm_diffnet == f0_gen._denoise_fn): tie them
    for net, gen in (("gm_diffnet", "f0_gen"), ("gm_diffnet_inpainte", "f0_gen_inpainte")):
        for k in list(sd.keys()):
            if k.startswith(gen + "._denoise_fn."):
                sd[k] = sd[net + "." + k[len(gen + "._denoise_fn."):]]
    if hp["f0_gen"] == "conv":
        # The generic init puts the predicted f0 (log2 Hz) around 0-3, i.e. below 8 Hz, where every frame falls into
        # coarse bin 1.  Centre the f0 row on 8 (256 Hz) with a spread of about +-0.7 octave so that f0_to_coarse and
        # pitch_embed see a realistic range; the uv row (about half the frames > 0) is left as generated.  No random
        # numbers are drawn here.
        for p in ("pitch_predictor.", "pitch_inpainter_predictor."):
            sd[p + "linear.weight"][0] *= 0.35
            sd[p + "linear.bias"][0] = 8.0
    return sd


def vocoder_state_dict(h=None, seed=0):
    h = dict(DEFAULT_VOCODER_CONFIG, **(h or {}))
    g = torch.Generator().manual_seed(seed + 7919)
    sd = OrderedDict()
    shapes = vocoder_param_shapes(h)
    # weight_g precedes weight_v in the reference's state_dict order but is derived from it:
    # visit the v tensors first (generation order is part of the seed contract), then the rest.
    order = [x for x in shapes if x[0].endswith("weight_v")] + [x for x in shapes if not x[0].endswith("weight_v")]
    for name, shape in order:
        base = name.split(".")[-1]
        if base == "weight_v":
            if name.startswith("ups."):  # ConvTranspose1d [Cin, Cout, k], stride u: fan_in = Cin*k/u
                i = int(name.split(".")[1])
                fan_in = shape[0] * shape[2] / h["upsample_rates"][i]
            else:
                fan_in = int(np.prod(shape[1:]))
            gain = 0.5 if name.startswith("conv_post") else 1.0
            t = torch.randn(shape, generator=g) * (gain / math.sqrt(fan_in))
        elif base == "weight_g":
            v = sd[name[:-1] + "v"]
            # weight_norm(dim=0): norm over dims != 0; keep the effective weight close to v
            nrm = v.reshape(v.shape[0], -1).norm(dim=1).reshape(shape)
            t = nrm * (1.0 + 0.05 * torch.randn(shape, generator=g))
        elif name.startswith("noise_convs") and base == "weight":
            t = torch.randn(shape, generator=g) / math.sqrt(shape[2])
        elif name == "m_source.l_linear.weight":
            t = torch.randn(shape, generator=g) * 1.5
        elif base == "bias":
            t = 0.05 * torch.randn(shape, generator=g)
        else:
            fan_in = int(np.prod(shape[1:]))
            t = torch.randn(shape, generator=g) / math.sqrt(fan_in)
        sd[name] = t.float().contiguous()
    return OrderedDict((n, sd[n]) for n, _ in shapes)


# ----------------------------------------------------------------------------------------------
# synthetic inputs (SURVEY.md §8d)
# ----------------------------------------------------------------------------------------------
def make_utterance(seconds, utt_idx=0, ref_frames=1125, frames=None, phones=None):
    """One synthetic utterance: dict of CPU tensors (no batch dim).

    txt_tokens int64 [P], note int64 [P], note_dur f32 [P], note_type int64 [P], mel2ph int64 [F]
    (1-based, even split), spk_embed/emo_embed f32 [256] (L2-normalised), ref_mels f32 [R,80],
    ref_f0 f32 [R] (log2 Hz, unvoiced frames interpolated like norm_interp_f0 does).
    """
    g = torch.Generator().manual_seed(1234 + utt_idx)
    F_ = int(round(187.5 * seconds)) if frames is None else int(frames)
    P = max(4, int(round(7.5 * seconds))) if phones is None else int(phones)
    txt = torch.randint(3, N_TOKENS, (P,), generator=g)
    note = torch.randint(48, 73, (P,), generator=g)
    rest = torch.rand(P, generator=g) < 0.1
    note = torch.where(rest, torch.zeros_like(note), note)
    note_type = torch.where(rest, torch.ones_like(note), torch.full_like(note, 2))
    note_dur = 0.1 + 0.5 * torch.rand(P, generator=g)
    # even split of F frames over P phones, 1-based
    bounds = torch.linspace(0, F_, P + 1).round().long()
    mel2ph = torch.zeros(F_, dtype=torch.long)
    for p in range(P):
        mel2ph[bounds[p]:bounds[p + 1]] = p + 1
    spk = torch.randn(256, generator=g)
    spk = spk / spk.norm()
    emo = torch.randn(256, generator=g)
    emo = emo / emo.norm()
    R = int(ref_frames)
    ref = (-3.0 + 0.8 * torch.randn(R, 80, generator=g)).clamp(-6.0, 0.6)
    ref[:, 0] = torch.where(ref[:, 0] == 0, torch.full_like(ref[:, 0], -1e-3), ref[:, 0])
    hz = 150.0 + 350.0 * torch.rand(R, generator=g)
    uv = torch.rand(R, generator=g) < 0.15
    uv[0] = False
    uv[-1] = False
    f0 = torch.log2(hz).numpy().astype(np.float64)
    uvn = uv.numpy()
    f0[uvn] = np.interp(np.where(uvn)[0], np.where(~uvn)[0], f0[~uvn])
    return {"txt_tokens": txt, "note": note, "note_dur": note_dur.float(), "note_type": note_type,
            "mel2ph": mel2ph, "spk_embed": spk.float(), "emo_embed": emo.float(),
            "ref_mels": ref.float(), "ref_f0": torch.from_numpy(f0).float(), "seconds": float(seconds)}


def batch_seconds(n, seed=1234, lo=2.0, hi=15.0):
    """Utterance durations of BASELINE.json configs 3/4: default_rng(1234).uniform(2,15,n)."""
    return np.random.default_rng(seed).uniform(lo, hi, n)


def make_batch(n, seed=1234, ref_frames=1125, first_idx=0):
    secs = batch_seconds(n, seed)
    return [make_utterance(float(s), utt_idx=first_idx + i, ref_frames=ref_frames) for i, s in enumerate(secs)]
