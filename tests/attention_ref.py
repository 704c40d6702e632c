"""Float64 restatement of key-padding-masked multi-head attention, the operation of both attention kernels
(csrc/attention.cu, csrc/attention_tc.cu): per utterance and per head of 128 columns,

    softmax((q * scale) k^T, masked keys -> -inf) v

A query row with no valid key (every key masked, or an utterance without keys) is NaN, as torch's softmax over a row of
-inf is.  The reference's FFT blocks (common_layers.py:277-286) and style aligner (lse.py:41) run this between their in-
and out-projections (oracle.stylesinger_oracle.mha); tests/test_attention_ref_cpu.py pins the two together."""
import torch

HD = 128


def attention(q, k, v, scale, keymask=None, heads=2):
    """One utterance: q [L, heads * 128], k and v [S, heads * 128], keymask [S] (0 = masked) or None -> float64
    [L, heads * 128]."""
    q, k, v = q.double(), k.double(), v.double()
    keep = torch.ones(k.shape[0], dtype=torch.bool) if keymask is None else torch.as_tensor(keymask) != 0
    out = torch.empty(q.shape[0], heads * HD, dtype=torch.float64)
    for h in range(heads):
        sl = slice(h * HD, (h + 1) * HD)
        s = ((q[:, sl] * scale) @ k[:, sl].t()).masked_fill(~keep[None], float("-inf"))
        m = s.max(dim=1, keepdim=True).values if s.shape[1] else torch.full((s.shape[0], 1), float("-inf"), dtype=s.dtype)
        p = torch.exp(s - m)  # a row of -inf gives -inf - -inf = NaN
        out[:, sl] = (p @ v[:, sl]) / p.sum(dim=1, keepdim=True)
    return out
