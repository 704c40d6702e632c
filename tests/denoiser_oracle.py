"""The diffusion denoisers and their reverse steps in float64, over the test oracle (oracle/stylesinger_oracle.py).

diffnet64 / ddiffnet64 run O.diffnet / O.ddiffnet on the state dict cast to float64 with the step t passed as a float64
tensor (an integer t would make the step embedding fp32, and F.linear then meets float64 weights); the frequency table
of the sinusoidal step embedding stays fp32, as the reference builds it.  mel_chain64 and f0_chain64 restate
O.mel_diffusion_sample (K_step steps on the T-step schedule) and O.f0_diffusion_sample step for
step in float64 on the reference's fp32 schedule buffers, and return what a GPU comparison needs beyond the final
sample: every x_t / z_t, the fraction of x0 predictions the clip changed, and the Gumbel margin of every UV decision.
The noise comes in the C ABI's injected-noise layout (include/stylesinger_b200.h) for one utterance and is handed out
as float64.  tests/test_denoiser_f64_cpu.py pins all four against the reference fixtures and the fp32 oracle."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import stylesinger_oracle as O
from tests.common import acoustic_sd64

F0_PREFIX = ("gm_diffnet.", "gm_diffnet_inpainte.")  # which = 1 / 2 of ssb_denoiser_eval, 0 / 1 of the F0 sampler


def _t64(t, B):
    return torch.full((B,), float(t), dtype=torch.float64)


def diffnet64(spec, t, cond, hp, sd64=None, prefix="postdiff.denoise_fn."):
    """DiffNet.forward in float64. spec [B,1,80,F], t int, cond [B,256,F] -> [B,1,80,F].  sd64 / prefix: a float64 state
    dict and the net's key prefix (default: the DiffSinger mel denoiser of acoustic_sd64())."""
    with torch.no_grad():
        return O.diffnet(spec.double(), _t64(t, spec.shape[0]), cond.double(),
                         acoustic_sd64() if sd64 is None else sd64, hp, p=prefix)


def ddiffnet64(f0, uv, t, cond, hp, prefix):
    """DDiffNet.forward in float64. f0 [B,1,F], uv int64 [B,F], t int, cond [B,256,F] -> [B,3,F]."""
    with torch.no_grad():
        return O.ddiffnet(f0.double(), uv.long(), _t64(t, f0.shape[0]), cond.double(), acoustic_sd64(), hp, prefix)


def _gauss64(T, K, max_beta):
    """The first K rows of the T-step schedule's fp32 buffers, as float64 (see O.k_step)."""
    return {k: v[:K].double() for k, v in O._gauss_tables(T, max_beta).items()}


def spec_bounds(hp):
    smin = torch.tensor(hp["spec_min"], dtype=torch.float32)[:hp["keep_bins"]].double()
    smax = torch.tensor(hp["spec_max"], dtype=torch.float32)[:hp["keep_bins"]].double()
    return smin, smax


def mel_chain64(cond, coarse, hp, K, noise):
    """DiffusionDecoder.forward(infer=True) from t = K (K_step) for one utterance, in float64.
    cond [F,256], coarse [F,80], noise [K+1, F, 80] (the q_sample draw, then one per step t = K-1 .. 0).
    Returns {"mel": [F,80], "x": [x_K, x_{K-1}, .., x_0] each [F,80] (normalised), "clip": per step t = K-1 .. 0 the
    fraction of x0 predictions with |x0| > 1}."""
    s = _gauss64(hp["timesteps"], K, hp["max_beta"])
    smin, smax = spec_bounds(hp)
    c = cond.double().t()[None]
    nz = noise.double()
    x = s["sqrt_alphas_cumprod"][K - 1] * ((coarse.double() - smin) / (smax - smin) * 2 - 1) + \
        s["sqrt_one_minus_alphas_cumprod"][K - 1] * nz[0]
    xs, clip = [x], []
    for i in reversed(range(K)):
        eps = diffnet64(x.t()[None, None], i, c, hp)[0, 0].t()
        x0 = s["sqrt_recip_alphas_cumprod"][i] * x - s["sqrt_recipm1_alphas_cumprod"][i] * eps
        clip.append(float((x0.abs() > 1.0).double().mean()))
        x0 = x0.clamp(-1.0, 1.0)
        mean = s["posterior_mean_coef1"][i] * x0 + s["posterior_mean_coef2"][i] * x
        x = mean + (0.0 if i == 0 else 1.0) * (0.5 * s["posterior_log_variance_clipped"][i]).exp() * nz[K - i]
        xs.append(x)
    return {"mel": (x + 1) / 2 * (smax - smin) + smin, "x": xs, "clip": clip}


def f0_chain64(cond, lo, hi, hp, prefix, gauss, unif):
    """GaussianMultinomialDiffusion.sample (O.f0_diffusion_sample) for one utterance, in float64.
    cond [256,F]; lo, hi [F] (O.midi_clip_band); gauss [T+1, F] (z_T, then one draw per step t = T-1 .. 0); unif
    [T, F, 2] (the Gumbel uniforms of step t = T-1 .. 0, class last).  The UV initialisation draw of the reference is
    not an input: its result is never read.
    Returns {"z": [z_T, .., z_0], "uv": [uv_T, .., uv_0] (int64 [F]), "margin": per step t = T-1 .. 0 the float64
    |(g1 + logp1) - (g0 + logp0)| of every frame, "clip": per step the fraction of x0 predictions outside [lo, hi]}."""
    T = hp["f0_timesteps"]
    s = _gauss64(T, T, hp["f0_max_beta"])
    m = {k: v.double() for k, v in O._multi_tables(T, hp["f0_max_beta"]).items()}
    c = cond.double()[None]
    lo, hi = lo.double(), hi.double()
    g64, u64 = gauss.double(), unif.double()
    Fr = c.shape[-1]
    ln2 = np.log(2)
    z = g64[0]
    uv = torch.zeros(Fr, dtype=torch.long)
    zs, uvs, margins, clip = [z], [uv], [], []
    for k, i in enumerate(reversed(range(T))):
        out = ddiffnet64(z[None, None], uv[None], i, c, hp, prefix)[0]
        eps, logits = out[0], out[1:][None]
        x0 = s["sqrt_recip_alphas_cumprod"][i] * z - s["sqrt_recipm1_alphas_cumprod"][i] * eps
        clip.append(float(((x0 < lo) | (x0 > hi)).double().mean()))
        x0 = torch.max(torch.min(x0, hi), lo)
        mean = s["posterior_mean_coef1"][i] * x0 + s["posterior_mean_coef2"][i] * z
        z = mean + (0.0 if i == 0 else 1.0) * (0.5 * s["posterior_log_variance_clipped"][i]).exp() * g64[k + 1]
        log_z = torch.log(F.one_hot(uv[None], 2).permute(0, 2, 1).double().clamp(min=1e-30))
        l0 = F.log_softmax(logits, dim=1)
        tm1 = max(i - 1, 0)
        ev = O._log_add_exp(l0 + m["log_cumprod_alpha"][tm1], m["log_1_min_cumprod_alpha"][tm1] - ln2)
        if i == 0:
            ev = l0
        un = ev + O._log_add_exp(log_z + m["log_alpha"][i], m["log_1_min_alpha"][i] - ln2)
        logp = (un - torch.logsumexp(un, dim=1, keepdim=True))[0]
        g = -torch.log(-torch.log(u64[k].t() + 1e-30) + 1e-30)
        v = g + logp
        margins.append((v[1] - v[0]).abs())
        uv = v.argmax(0)
        zs.append(z)
        uvs.append(uv)
    return {"z": zs, "uv": uvs, "margin": margins, "clip": clip}
