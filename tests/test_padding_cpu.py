"""Pin the oracle's padding masks against the unmodified reference (tools/make_golden.py padded): padding phones
(txt_tokens == 0), an interior and a trailing run of padding frames (mel2ph == 0), and a reference mel with all-zero
trailing rows plus one row whose column 0 alone is 0."""
import numpy as np

from tests.common import golden, hp_for, oracle_forward, utt_from_fixture

TOL = 2e-5  # fp32 CPU, same op order up to BLAS blocking


def _maxabs(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max())


def test_fixture_has_every_kind_of_padding():
    g, meta = golden("ref_padded_T4")
    u = utt_from_fixture(g)
    assert (u["txt_tokens"][-3:] == 0).all() and (u["txt_tokens"][:-3] > 0).all()
    m = u["mel2ph"].numpy()
    pad = np.flatnonzero(m == 0)
    assert pad[-1] == len(m) - 1 and np.any(np.diff(pad) > 1)  # a trailing run and an interior one
    ref = u["ref_mels"].numpy()
    col0 = ref[:, 0] == 0
    row = np.abs(ref).sum(1) == 0
    assert row[-8:].all() and (u["ref_f0"][-8:] == 0).all()
    assert np.any(col0 & ~row)  # column 0 masks this row, the whole-row mask does not


def test_padded_forward_matches_reference():
    g, meta = golden("ref_padded_T4")
    r, ns = oracle_forward(utt_from_fixture(g), hp_for(meta["T"]), meta["seed"])
    assert [[k, list(sh)] for k, sh in ns.log] == meta["noise_log"]  # same RNG draw sequence
    assert np.array_equal(r["rq_codes"][0].numpy(), g["rq_codes"])
    for k in ["style", "pitch_pred", "decoder_inp", "coarse_mel", "mel_out"]:
        assert _maxabs(r[k][0].numpy(), g[k]) < TOL, k
    assert _maxabs(r["f0_denorm"][0].numpy(), g["f0_denorm"]) < 1e-3  # Hz
    assert (g["f0_denorm"][g["in_mel2ph"] == 0] == 0).all()


def test_padded_duration_path_matches_reference():
    g, meta = golden("ref_padded_T4")
    r, ns = oracle_forward(utt_from_fixture(g), hp_for(meta["T"]), meta["seed"] + 1, use_mel2ph=False)
    assert [[k, list(sh)] for k, sh in ns.log] == meta["dur_noise_log"]
    assert np.array_equal(r["mel2ph"][0].numpy(), g["dur_mel2ph"])  # integer path: exact
    assert _maxabs(r["dur"][0].numpy(), g["dur_logdur"]) < TOL
    assert _maxabs(r["mel_out"][0].numpy(), g["dur_mel_out"]) < TOL
    assert _maxabs(r["f0_denorm"][0].numpy(), g["dur_f0_denorm"]) < 1e-3
