"""The ProDiff and PLMS mel samplers in float64, over the test oracle (oracle/stylesinger_oracle.py).

prodiff_chain64 restates ProDiffusion.forward(infer=True) (prodiff.py:204-222) and plms_chain64 the pndm_speedup loop of
GaussianDiffusion.forward from t = K_step (shallow_diffusion_tts.py:164-197,244-260) step by step in float64, on the
reference's fp32 schedule buffers, through denoiser_oracle.diffnet64 on the model's state dict cast to float64.  Besides
the final mel they return what a GPU comparison needs to tell where an error grows: every x_t, every denoiser input and
output, and for PLMS the history order each step used.  Noise comes in the C ABI's injected-noise layout
(include/stylesinger_b200.h) for one utterance; equal-length utterances can run as one float64 batch.
tests/test_sampler_f64_cpu.py pins both against the reference fixtures and the fp32 oracles."""
import torch

from oracle import stylesinger_oracle as O
from tests import denoiser_oracle as DO
from tests.common import prodiff_sd

_C = {}


def prodiff_sd64():
    if "sd64" not in _C:
        _C["sd64"] = {k: (v.double() if v.is_floating_point() else v) for k, v in prodiff_sd().items()}
    return _C["sd64"]


def _eval(x, t, c, hp, sd64=None, prefix="postdiff.denoise_fn."):
    """One denoiser evaluation on x [B,F,80] with c [B,256,F] -> [B,F,80]."""
    return DO.diffnet64(x.transpose(1, 2)[:, None], t, c, hp, sd64, prefix)[:, 0].transpose(1, 2)


def _one(r):
    """A chain's result for a batch of one utterance, without the batch dimension."""
    def strip(w):
        if isinstance(w, tuple):
            return w[0], w[1][0]
        return w[0] if isinstance(w, torch.Tensor) else w
    return {k: (v[0] if isinstance(v, torch.Tensor) else [strip(w) for w in v]) for k, v in r.items()}


def _prodiff_chain64(cond, hp, noise):
    """ProDiffusion.forward(cond, infer=True) for B utterances of one length, in float64.  cond [B,F,256] (decoder_inp);
    noise [T+1, B, F, 80] (x_T, then one draw per step t = T-1 .. 0; the last is drawn but multiplied by 0).
    x_T = noise[0]; per step x0 = denoise_fn(x_t, t, cond) with no eps conversion and no clip, then the posterior mean
    plus exp(0.5 logvar) noise; denorm_spec is the identity.
    Returns {"mel": [B,F,80], "x": [x_T, .., x_0], "x0": per step t = T-1 .. 0 the denoiser output}."""
    T = hp["timesteps"]
    s = {k: v.double() for k, v in O.prodiff_tables(T).items()}
    c = cond.double().transpose(1, 2)
    nz = noise.double()
    x = nz[0]
    xs, x0s = [x], []
    for k, i in enumerate(reversed(range(T))):
        x0 = _eval(x, i, c, hp, prodiff_sd64(), O.PRODIFF_PREFIX)
        x0s.append(x0)
        mean = s["posterior_mean_coef1"][i] * x0 + s["posterior_mean_coef2"][i] * x
        x = mean + (0.0 if i == 0 else 1.0) * (0.5 * s["posterior_log_variance_clipped"][i]).exp() * nz[k + 1]
        xs.append(x)
    return {"mel": x, "x": xs, "x0": x0s}


def prodiff_chain64(cond, hp, noise):
    """_prodiff_chain64 for one utterance (cond [F,256], noise [T+1, F, 80]: the C ABI's layout) or, with cond [B,F,256]
    and noise [T+1, B, F, 80], for B utterances of one length as one float64 batch."""
    if cond.dim() == 3:
        return _prodiff_chain64(cond, hp, noise)
    return _one(_prodiff_chain64(cond[None], hp, noise[:, None]))


def plms_steps(K, interval):
    """The step numbers of the pndm_speedup loop from t = K: reversed(range(0, K, interval))."""
    return list(reversed(range(0, K, interval)))


def _plms_chain64(cond, coarse, hp, K, interval, q_noise):
    """GaussianDiffusion.forward(infer=True) with pndm_speedup = interval from t = K (K_step), for B utterances of one
    length, in float64.  cond [B,F,256], coarse [B,F,80], q_noise [B,F,80] (the one draw: q_sample of norm_spec(coarse)
    at K-1).
    Each step t evaluates eps at x_t; the first (an empty history) also evaluates eps at the trial point
    x_pred(x_t, eps, t) and step max(t - interval, 0) and averages the two; later steps extrapolate with the
    Adams-Bashforth weights of the 1 to 3 newest history entries.  x_{t-interval} = x_pred(x_t, prime, t) with
    alphas_cumprod at t and at max(t - interval, 0).
    Returns {"mel": [B,F,80], "x": [x_K, then x after each step], "eps": per step the un-extrapolated eps,
    "calls": every denoiser evaluation as (t, input x), "order": per step the number of history entries used (0: the
    second-order start)}."""
    T = hp["timesteps"]
    s = DO._gauss64(T, K, hp["max_beta"])
    ac = s["alphas_cumprod"]
    smin, smax = DO.spec_bounds(hp)
    c = cond.double().transpose(1, 2)
    x = s["sqrt_alphas_cumprod"][K - 1] * ((coarse.double() - smin) / (smax - smin) * 2 - 1) + \
        s["sqrt_one_minus_alphas_cumprod"][K - 1] * q_noise.double()

    def x_pred(x, e, t):  # get_x_pred (shallow_diffusion_tts.py:170-178)
        a_t, a_prev = ac[t], ac[max(t - interval, 0)]
        a_t_sq, a_prev_sq = a_t.sqrt(), a_prev.sqrt()
        return x + (a_prev - a_t) * (x / (a_t_sq * (a_t_sq + a_prev_sq))
                                     - e / (a_t_sq * (((1 - a_prev) * a_t).sqrt() + ((1 - a_t) * a_prev).sqrt())))

    xs, epss, calls, orders, hist = [x], [], [], [], []
    for t in plms_steps(K, interval):
        calls.append((t, x))
        eps = _eval(x, t, c, hp)
        orders.append(len(hist))
        if not hist:
            xp = x_pred(x, eps, t)
            tp = max(t - interval, 0)
            calls.append((tp, xp))
            prime = (eps + _eval(xp, tp, c, hp)) / 2
        elif len(hist) == 1:
            prime = (3 * eps - hist[-1]) / 2
        elif len(hist) == 2:
            prime = (23 * eps - 16 * hist[-1] + 5 * hist[-2]) / 12
        else:
            prime = (55 * eps - 59 * hist[-1] + 37 * hist[-2] - 9 * hist[-3]) / 24
        x = x_pred(x, prime, t)
        hist = (hist + [eps])[-3:]
        xs.append(x)
        epss.append(eps)
    return {"mel": (x + 1) / 2 * (smax - smin) + smin, "x": xs, "eps": epss, "calls": calls, "order": orders}


def plms_chain64(cond, coarse, hp, K, interval, q_noise):
    """_plms_chain64 for one utterance (cond [F,256], coarse and q_noise [F,80]) or, with a leading dimension B on all
    three, for B utterances of one length as one float64 batch."""
    if cond.dim() == 3:
        return _plms_chain64(cond, coarse, hp, K, interval, q_noise)
    return _one(_plms_chain64(cond[None], coarse[None], hp, K, interval, q_noise[None]))


def plms_evals(K, interval):
    """Denoiser evaluations of one PLMS call: one per step, plus the first step's second."""
    return len(plms_steps(K, interval)) + 1
