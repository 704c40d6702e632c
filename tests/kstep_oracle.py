"""Shallow diffusion (hparams['K_step'] < timesteps) over the test oracle (oracle/stylesinger_oracle.py).

GaussianDiffusion.__init__ builds its buffers for the full `timesteps`-long schedule and stores K_step beside them
(shallow_diffusion_tts.py:68-119); DiffusionDecoder.forward(infer=True) then draws x_K = q_sample(norm_spec(coarse), K-1)
and runs the K reverse steps t = K-1 .. 0 (:297-304), and the PLMS loop starts from the same t = K (:244-260).  Every
index the samplers read is below K, so a K-step run on the T-step schedule is the oracle's own sampler run with
timesteps = K over the first K entries of the T-step tables.  That is what these wrappers do: the sampler code stays the
one tests/test_oracle_golden.py pins, and tests/test_kstep_cpu.py pins these wrappers against the unmodified reference
(tests/golden/ref_kstep.npz)."""
import contextlib

from oracle import stylesinger_oracle as O


def k_step(hp):
    return int(hp.get("K_step", hp["timesteps"]))


@contextlib.contextmanager
def _first_k_of_schedule(T, K):
    full = O._gauss_tables

    def tables(n, max_beta):
        assert n == K, (n, K)
        return {k: v[:K] for k, v in full(T, max_beta).items()}

    O._gauss_tables = tables
    try:
        yield
    finally:
        O._gauss_tables = full


def mel_diffusion_sample(cond, coarse_mel, sd, hp, noise, return_steps=False):
    """DiffusionDecoder.forward(infer=True) with t = hp['K_step']: K + 1 draws (q_sample, then one per step)."""
    T, K = hp["timesteps"], k_step(hp)
    with _first_k_of_schedule(T, K):
        return O.mel_diffusion_sample(cond, coarse_mel, sd, dict(hp, timesteps=K), noise, return_steps)


def mel_diffusion_sample_plms(cond, coarse_mel, sd, hp, noise, interval):
    """The pndm_speedup loop from t = hp['K_step']: reversed(range(0, K, interval)), one draw (q_sample at K-1)."""
    T, K = hp["timesteps"], k_step(hp)
    with _first_k_of_schedule(T, K):
        return O.mel_diffusion_sample_plms(cond, coarse_mel, sd, dict(hp, timesteps=K), noise, interval)


def stylesinger_forward(sd, hp, txt_tokens, note, note_dur, note_type, spk_embed, emo_embed, ref_mels, ref_f0, noise, **kw):
    """O.stylesinger_forward with the mel sampler above: the same draws in the same order, the mel sampler's last."""
    r = O.stylesinger_forward(sd, hp, txt_tokens, note, note_dur, note_type, spk_embed, emo_embed, ref_mels, ref_f0, noise,
                              skip_diffusion=True, **kw)
    r["mel_out"] = mel_diffusion_sample(r["diff_cond"], r["coarse_mel"], sd, hp, noise)
    return r
