"""The per-utterance (keyed) Philox draw plan in NumPy, built from tests/philox_ref.py: utterance b of a keyed call draws
with key seeds[b] and counts its own rows from 0 (include/stylesinger_b200.h, csrc/philox.cuh).  Each builder lays the
draws out the way the C ABI takes injected noise, so a keyed call can be compared with a run that injects its plan.
Test-only: nothing here imports the package under test."""
import numpy as np

from tests import philox_ref as P


def _per_utt(seeds, frame_offsets, one):
    """Concatenate, along the tight axis, one(seed_b, [0, len_b]) of every utterance; the tight axis is axis 1 of
    the blocks `one` returns."""
    fo = np.asarray(frame_offsets)
    parts = [one(int(seeds[b]), np.array([0, fo[b + 1] - fo[b]])) for b in range(len(fo) - 1)]
    return np.concatenate(parts, axis=1)


def mel_noise(seeds, T, frame_offsets, steps=None):
    """[(T+1), sumF, 80]: utterance b's rows are philox_ref.mel_noise(seeds[b], T, [0, len_b])."""
    return _per_utt(seeds, frame_offsets, lambda s, o: P.mel_noise(s, T, o, steps))


def f0_gauss_noise(seeds, net, T, frame_offsets):
    return _per_utt(seeds, frame_offsets, lambda s, o: P.f0_gauss_noise(s, net, T, o))


def f0_unif_noise(seeds, net, T, frame_offsets):
    return _per_utt(seeds, frame_offsets, lambda s, o: P.f0_unif_noise(s, net, T, o))


def vocoder_rand_ini(seeds):
    """[B, 9]: every utterance reads stream_voc_ini(0) under its own key."""
    return np.concatenate([P.vocoder_rand_ini(int(s), 1) for s in seeds], axis=0)


def vocoder_src_noise(seeds, frame_offsets, hop=256):
    fo = np.asarray(frame_offsets)
    return np.concatenate([P.vocoder_src_noise(int(seeds[b]), np.array([0, fo[b + 1] - fo[b]]), hop)
                           for b in range(len(fo) - 1)], axis=0)


def acoustic_noise(seeds, T_mel, T_f0, frame_offsets):
    """The injected-noise dict of AcousticModel.forward that a keyed forward draws."""
    return {"f0_gauss": [f0_gauss_noise(seeds, n, T_f0, frame_offsets) for n in range(2)],
            "f0_unif": [f0_unif_noise(seeds, n, T_f0, frame_offsets) for n in range(2)],
            "mel": mel_noise(seeds, T_mel, frame_offsets)}
