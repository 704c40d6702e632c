"""Pins tests/attention_ref.py, the float64 arbiter of both attention kernels, to the oracle's multi-head attention
(oracle.stylesinger_oracle.mha with identity projections) and to torch's scaled_dot_product_attention, in float64."""
import pytest
import torch
import torch.nn.functional as F

from oracle import stylesinger_oracle as O
from tests import attention_ref as A

SCALE = 128 ** -0.5


def _qkv(L, S, seed, sigma=1.5, heads=2):
    g = torch.Generator().manual_seed(seed)
    E = heads * 128
    q = torch.randn(L, E, generator=g, dtype=torch.float64) * sigma
    k = torch.randn(S, E, generator=g, dtype=torch.float64) * sigma
    v = torch.randn(S, E, generator=g, dtype=torch.float64)
    return q, k, v


@pytest.mark.parametrize("sigma", [1.5, 6.0])
def test_matches_oracle_mha_with_identity_projections(sigma):
    """A batch of two utterances padded to one key length, the shorter one's padding keys masked, as the reference
    batches them; the second utterance also masks two of its own keys."""
    E, L, S = 256, 37, 70
    eye = torch.eye(E, dtype=torch.float64)
    q, k, v = _qkv(2 * L, 2 * S, 5, sigma)
    q, k, v = q.reshape(2, L, E), k.reshape(2, S, E), v.reshape(2, S, E)
    pad = torch.zeros(2, S, dtype=torch.bool)
    pad[0, 51:] = True
    pad[1, [0, 64]] = True
    with torch.no_grad():
        o = O.mha(q.transpose(0, 1), k.transpose(0, 1), v.transpose(0, 1), torch.cat([eye, eye, eye]), None, eye, None,
                  num_heads=2, key_padding_mask=pad).transpose(0, 1)
    for b in range(2):
        r = A.attention(q[b], k[b], v[b], SCALE, keymask=(~pad[b]).double())
        assert torch.allclose(r, o[b], rtol=1e-12, atol=1e-12), b
    # the shorter utterance alone, without its padding keys, is the same thing
    assert torch.allclose(A.attention(q[0], k[0, :51], v[0, :51], SCALE), o[0], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("heads,L,S,scale,sigma", [(2, 1, 1, SCALE, 1.5), (2, 65, 320, SCALE, 1.5), (1, 9, 129, SCALE, 6.0),
                                                   (2, 64, 57, 0.3, 1.5), (2, 3, 2812, SCALE, 1.5)])
def test_matches_scaled_dot_product_attention(heads, L, S, scale, sigma):
    q, k, v = _qkv(L, S, L + S, sigma, heads)
    g = torch.Generator().manual_seed(S)
    keep = torch.rand(S, generator=g) > 0.3
    keep[S // 2] = True
    for mask in (None, keep.double()):
        r = A.attention(q, k, v, scale, keymask=mask, heads=heads)
        split = [t.reshape(t.shape[0], heads, 128).transpose(0, 1)[None] for t in (q, k, v)]
        am = None if mask is None else keep[None, None, None, :]
        ref = F.scaled_dot_product_attention(*split, attn_mask=am, scale=scale)[0].transpose(0, 1).reshape(L, heads * 128)
        assert torch.allclose(r, ref, rtol=1e-11, atol=1e-12), (heads, L, S, mask is None)


def test_rows_without_a_valid_key_are_nan():
    q, k, v = _qkv(5, 9, 1)
    assert torch.isnan(A.attention(q, k[:0], v[:0], SCALE)).all()
    assert torch.isnan(A.attention(q, k, v, SCALE, keymask=torch.zeros(9))).all()
    one = torch.zeros(9)
    one[4] = 1
    r = A.attention(q, k, v, SCALE, keymask=one)  # one valid key: its value row, whatever the scores
    assert torch.allclose(r, v[4].expand(5, -1), rtol=0, atol=1e-15)


def test_flat_scores_average_the_values():
    _, k, v = _qkv(1, 2812, 2)
    r = A.attention(torch.zeros(3, 256, dtype=torch.float64), k, v, SCALE)
    assert torch.allclose(r, v.mean(0).expand(3, -1), rtol=0, atol=1e-14)
