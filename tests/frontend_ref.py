"""The reference-audio front-end in float64, with per-element error bounds for the CUDA kernels that compute it.

The mel spectrogram (ssb_melspec_*) is restated on oracle/frontend_oracle.py's pieces (the periodic Hann window, np.pad
centring, the Slaney filterbank) but kept in float64 to the end, so that what the kernel is compared with carries no fp32
rounding of its own.  The kernel computes the windowed DFT as ONE fp32 GEMM with K = n_fft (the window folded into the
weights), so the rounding of a bin is bounded by the frame's windowed L1 norm S_f = sum_j |w_j x_j|, not by the bin's
own magnitude: a quiet band under a loud one is only as accurate as the loud one allows.  Per element:

    |d |X_k||   <= alpha S_f
    |d mel_i|   <= alpha S_f sum_k M_ik + beta (M |X|)_i                          (|X|, librosa_wav2spec)
    |d pmel_i|  <= alpha S_f sum_k M_ik (2 |X_k| + alpha S_f) + beta (M |X|^2)_i  (|X|^2, librosa.feature.melspectrogram)

alpha covers the DFT GEMM and the fp32 rounding of its weights, beta the magnitude, the mel GEMM (all terms positive, so
relative to its result) and the fp32 rounding of the filterbank.  In log mode the linear bound is pushed through
log10(max(eps, .)): the output must lie between log10(max(eps, v - d)) and log10(max(eps, v + d)), widened by the
rounding of log10f itself, so a value within the bound of eps may land anywhere between the two sides of the floor.

The LSTM half (ssb_lstm_encoder_*) is oracle.frontend_oracle.lstm_hidden in float64 with an overflow-free sigmoid: the
emotion encoder's inputs are power mels of order 1e2 and more, whose gate pre-activations overflow np.exp(-x).
"""
import numpy as np

from oracle import frontend_oracle as FO

# name -> MelSpectrogram arguments and the geometry the reference computes with
CONFIGS = {
    # librosa_wav2spec of egs/stylesinger.yaml: zero centring, |X|, log10(max(eps, .))
    "wav2spec": dict(sr=48000, n_fft=1024, hop=256, win=1024, n_mels=80, fmin=20.0, fmax=24000.0, eps=1e-6,
                     reflect=False, power=False, log=True),
    # the same geometry without the log: a wrong value cannot hide under the floor
    "wav2spec_lin": dict(sr=48000, n_fft=1024, hop=256, win=1024, n_mels=80, fmin=20.0, fmax=24000.0, eps=1e-6,
                         reflect=False, power=False, log=False),
    # the emotion / speaker encoders' features (data_gen/tts/emotion/audio.py): reflect centring, |X|^2, no log
    "emotion": dict(sr=16000, n_fft=400, hop=160, win=400, n_mels=40, fmin=0.0, fmax=8000.0, eps=1e-6,
                    reflect=True, power=True, log=False),
}


def melspec(cfg, device):
    """The CUDA front-end of a configuration."""
    from stylesinger_b200.engine import MelSpectrogram
    c = CONFIGS[cfg]
    hp = dict(audio_sample_rate=c["sr"], fft_size=c["n_fft"], hop_size=c["hop"], win_size=c["win"], audio_num_mel_bins=c["n_mels"],
              fmin=c["fmin"], fmax=c["fmax"])
    return MelSpectrogram(hp, device, eps=c["eps"], pad_reflect=c["reflect"], power=c["power"], log=c["log"])


def spectrum64(y, cfg):
    """|X| [T, 1 + n_fft / 2] in float64 of librosa.stft(center=True) and the frames' windowed L1 norms S [T]."""
    c = CONFIGS[cfg]
    n_fft, hop = c["n_fft"], c["hop"]
    w = FO.pad_center(FO.hann_periodic(c["win"]), n_fft)
    yp = np.pad(np.asarray(y, np.float32).astype(np.float64), n_fft // 2, mode="reflect" if c["reflect"] else "constant")
    frames = np.lib.stride_tricks.sliding_window_view(yp, n_fft)[::hop] * w
    return np.abs(np.fft.rfft(frames, axis=1)), np.abs(frames).sum(axis=1)


def _basis64(cfg):
    c = CONFIGS[cfg]
    return FO.mel_basis(c["sr"], c["n_fft"], c["n_mels"], c["fmin"], c["fmax"]).astype(np.float64)


def reference(y, cfg, alpha, beta):
    """float64 reference of the configuration's output [T, n_mels] and the interval [lo, hi] the kernel's fp32 output must
    lie in (before the log10f rounding allowance of check()).  Also returns the two terms of the linear bound, A (the
    coefficient of alpha) and B (of beta), for calibration."""
    c = CONFIGS[cfg]
    M = _basis64(cfg)
    X, S = spectrum64(y, cfg)
    if c["power"]:
        v = (X * X) @ M.T
        A = S[:, None] * ((2.0 * X + alpha * S[:, None]) @ M.T)
    else:
        v = X @ M.T
        A = S[:, None] * M.sum(axis=1)[None, :]
    B = v
    d = alpha * A + beta * B
    if not c["log"]:
        return v, v - d, v + d, A, B
    eps = c["eps"]
    return (np.log10(np.maximum(eps, v)), np.log10(np.maximum(eps, v - d)), np.log10(np.maximum(eps, v + d)), A, B)


def check(out, y, cfg, alpha, beta):
    """Largest err / allowed of a kernel output against the float64 reference, and (A, B, err) for calibration.
    err / allowed <= 1 means the output lies inside the bound."""
    c = CONFIGS[cfg]
    out = np.asarray(out, np.float64)
    ref, lo, hi, A, B = reference(y, cfg, alpha, beta)
    assert out.shape == ref.shape, (out.shape, ref.shape)
    # log10f is accurate to 2 ulp (CUDA C Programming Guide, table of single-precision functions): 4 ulp of the result
    tau = 4.0 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64) if c["log"] else 0.0
    err = np.abs(out - ref)
    allowed = np.where(out >= ref, hi - ref, ref - lo) + tau
    ratio = np.divide(err, allowed, out=np.where(err > 0, np.inf, 0.0), where=allowed > 0)
    return float(ratio.max()) if ratio.size else 0.0, (A, B, np.abs(out - ref) if not c["log"] else None)


def calibrate(A, B, err):
    """Smallest (alpha, beta) for which err <= alpha A + beta B holds on these elements: alpha from the elements whose
    band is quiet against its frame (B <= A / 64, where the DFT's rounding dominates), beta from the rest given that alpha."""
    quiet = (B <= A / 64) & (A > 0)
    a = float(np.max(err[quiet] / A[quiet], initial=0.0)) if quiet.any() else 0.0
    loud = ~quiet & (B > 0)
    b = float(np.max((err[loud] - a * A[loud]) / B[loud], initial=0.0)) if loud.any() else 0.0
    return a, max(b, 0.0)


# ---- signals -------------------------------------------------------------------------------------------------------------
KINDS = ("sweep", "zeros", "gaps", "square", "impulse0", "impulse_end", "impulse_hop", "dc", "quiet4", "quiet8", "noise",
         "nyquist", "f16")


def _sweep(n, sr, rng):
    t = np.arange(n) / sr
    f0 = 180 + 120 * np.sin(2 * np.pi * 0.7 * t)
    y = sum(0.25 / k * np.sin(2 * np.pi * k * np.cumsum(f0) / sr) for k in range(1, 9))
    return y + 0.01 * rng.standard_normal(n)


def signal(kind, n, sr, hop, seed=0):
    """float32 test signal of n samples (kind 'f16' returns the float16 array the reference hands to the front-end)."""
    rng = np.random.default_rng(seed)
    y = np.zeros(n, np.float64)
    if kind == "sweep":
        y = _sweep(n, sr, rng)
    elif kind == "gaps":  # voiced segments with hard onsets between exact-zero pauses, and a few noise bursts (consonants)
        y = _sweep(n, sr, rng)
        gate = np.zeros(n)
        i = int(rng.integers(0, max(1, sr // 20)))
        while i < n:
            on = int(rng.integers(sr // 20, sr // 3))
            gate[i:i + on] = 1.0
            i += on + int(rng.integers(sr // 40, sr // 4))
        burst = (rng.random(n) < 2e-4).astype(np.float64)
        burst = np.convolve(burst, np.ones(sr // 100))[:n] * 0.3 * rng.standard_normal(n)
        y = y * gate + burst * (1 - gate)
    elif kind == "square":  # full-scale, clipped: every sample is exactly +-1
        y = np.where(np.sin(2 * np.pi * 440.0 * np.arange(n) / sr) >= 0, 1.0, -1.0)
    elif kind == "impulse0":
        if n:
            y[0] = 1.0
    elif kind == "impulse_end":
        if n:
            y[n - 1] = 1.0
    elif kind == "impulse_hop":
        if n:
            y[min(n - 1, hop * max(1, n // (2 * hop)))] = 1.0
    elif kind == "dc":  # all energy in the DC bin
        y[:] = 0.5
    elif kind == "quiet4":
        y = 1e-4 * _sweep(n, sr, rng)
    elif kind == "quiet8":
        y = 1e-8 * _sweep(n, sr, rng)
    elif kind == "noise":
        y = 0.3 * rng.standard_normal(n)
    elif kind == "nyquist":  # all energy in the Nyquist bin
        y = 0.5 * (1.0 - 2.0 * (np.arange(n) % 2))
    elif kind == "f16":
        return _sweep(n, sr, rng).astype(np.float16)
    elif kind != "zeros":
        raise ValueError(kind)
    return y.astype(np.float32)


# ---- the LSTM encoder in float64 ------------------------------------------------------------------------------------------
def _sigmoid(x):
    return 0.5 * (1.0 + np.tanh(0.5 * x))  # = 1 / (1 + exp(-x)) without overflow for large |x|


def lstm_hidden64(frames, sd, layers=FO.EMO_LAYERS):
    """FO.lstm_hidden (EmotionEncoder.inference) kept in float64 to the end: [P, H]."""
    x = np.asarray(frames, np.float64)
    P, T, _ = x.shape
    for l in range(layers):
        wih = sd["lstm.weight_ih_l%d" % l].astype(np.float64)
        whh_t = np.ascontiguousarray(sd["lstm.weight_hh_l%d" % l].astype(np.float64).T)
        b = sd["lstm.bias_ih_l%d" % l].astype(np.float64) + sd["lstm.bias_hh_l%d" % l].astype(np.float64)
        H = whh_t.shape[0]
        h = np.zeros((P, H))
        c = np.zeros((P, H))
        out = np.empty((P, T, H))
        xp = x @ wih.T + b
        for t in range(T):
            g = xp[:, t] + h @ whh_t
            c = _sigmoid(g[:, H:2 * H]) * c + _sigmoid(g[:, :H]) * np.tanh(g[:, 2 * H:3 * H])
            h = _sigmoid(g[:, 3 * H:]) * np.tanh(c)
            out[:, t] = h
        x = out
    return x[:, -1]


def embeds64(hidden, sd):
    """EmotionEncoder.forward after the LSTM: relu(linear(h)) L2-normalised per row, float64."""
    e = np.maximum(0.0, np.asarray(hidden, np.float64) @ sd["linear.weight"].astype(np.float64).T + sd["linear.bias"].astype(np.float64))
    return e / np.linalg.norm(e, axis=1, keepdims=True)


def utt_embed64(hidden):
    """Normalised mean of a group of partials' hidden states, float64."""
    raw = np.asarray(hidden, np.float64).mean(axis=0)
    return raw / np.linalg.norm(raw)
