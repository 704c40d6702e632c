"""HifiGanGenerator.forward after remove_weight_norm for every published layout: ResBlock1 (V1, V2) goes through the
project's oracle (oracle.stylesinger_oracle.hifigan_generator) unchanged; ResBlock2 (V3, hifigan_nsf.py:69-90) is
written out here in the same form, in fp32 or float64.  tests/test_vocoder_layouts_cpu.py pins both against the
reference's own generator (tests/golden/ref_vocoder_layouts.npz)."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from stylesinger_b200.hparams import HIFIGAN_V2, HIFIGAN_V3

# the layouts of tools/make_golden.py vocoder_layouts: V3 without NSF is the generator the `HifiGAN` registry class
# builds from a config without the harmonic source
LAYOUTS = {"v2": HIFIGAN_V2, "v3": HIFIGAN_V3, "v3_nonsf": dict(HIFIGAN_V3, use_pitch_embed=False)}

_SD = {}


def state_dict(name):
    if name not in _SD:
        _SD[name] = synth.vocoder_state_dict(LAYOUTS[name], seed=0)
    return _SD[name]


def hifigan_generator(mel, f0, sd, h, noise, dtype=torch.float32):
    """mel [B,80,F], f0 [B,F] or None -> wav [B,1,hop*F] in `dtype` (the NSF source stays fp32, see the oracle)."""
    if str(h.get("resblock", "1")) == "1":
        return O.hifigan_generator(mel, f0, sd, h, noise, dtype)
    rates, ks = h["upsample_rates"], h["upsample_kernel_sizes"]
    nk = len(h["resblock_kernel_sizes"])
    W = lambda n: O.fold_weight_norm(sd[n + ".weight_g"], sd[n + ".weight_v"]).to(dtype)
    P = lambda n: sd[n].to(dtype)
    har = None
    if f0 is not None:
        up = f0[:, None].repeat_interleave(int(np.prod(rates)), dim=2).transpose(1, 2)
        har = O.source_module(up, sd, noise).transpose(1, 2).to(dtype)
    x = F.conv1d(mel.to(dtype), W("conv_pre"), P("conv_pre.bias"), padding=3)
    for i, (u, k) in enumerate(zip(rates, ks)):
        x = F.leaky_relu(x, 0.1)
        x = F.conv_transpose1d(x, W(f"ups.{i}"), P(f"ups.{i}.bias"), stride=u, padding=(k - u) // 2)
        if har is not None:
            if i + 1 < len(rates):
                s = int(np.prod(rates[i + 1:]))
                x = x + F.conv1d(har, P(f"noise_convs.{i}.weight"), P(f"noise_convs.{i}.bias"), stride=s, padding=s // 2)
            else:
                x = x + F.conv1d(har, P(f"noise_convs.{i}.weight"), P(f"noise_convs.{i}.bias"))
        xs = None
        for j, (rk, rd) in enumerate(zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"])):
            r = x
            q = f"resblocks.{i * nk + j}."
            for m_, d in enumerate(rd[:2]):  # ResBlock2 builds two convs from dilation[0], dilation[1]
                xt = F.leaky_relu(r, 0.1)
                xt = F.conv1d(xt, W(f"{q}convs.{m_}"), P(f"{q}convs.{m_}.bias"), padding=(rk * d - d) // 2, dilation=d)
                r = xt + r
            xs = r if xs is None else xs + r
        x = xs / nk
    x = F.leaky_relu(x)  # default slope 0.01 (hifigan_nsf.py:165)
    x = F.conv1d(x, W("conv_post"), P("conv_post.bias"), padding=3)
    return torch.tanh(x)


def spec2wav(mel, f0, sd, h, noise, dtype=torch.float32):
    """mel np [F,80], f0 np [F] or None -> wav np [hop*F] (HifiGAN.spec2wav, B = 1)."""
    c = torch.from_numpy(np.ascontiguousarray(mel)).float().unsqueeze(0).transpose(2, 1)
    f = None if f0 is None else torch.from_numpy(np.ascontiguousarray(f0)).float()[None, :]
    with torch.no_grad():
        return hifigan_generator(c, f, sd, h, noise, dtype).view(-1).numpy()
