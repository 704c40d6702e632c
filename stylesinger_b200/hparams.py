"""Resolved hyper-parameters of the hot path.

Mirrors what the reference's ``set_hparams('egs/stylesinger.yaml')`` resolves to
(reference: egs/stylesinger.yaml:1-143, egs/egs_bases/tts/fs2.yaml, egs/egs_bases/tts/base.yaml;
loader utils/hparams.py:25-124).  The engine reads the same keys as the reference, so a
reference ``hparams`` dict can be passed in unchanged; keys it does not contain fall back to
these defaults.  HiFi-GAN architecture keys are NOT in the reference tree (they live in the
downloaded ``checkpoints/hifigan/config.yaml``, reference tasks/tts/vocoder_infer/hifigan_nsf.py:48-60);
``DEFAULT_VOCODER_CONFIG`` is the HiFi-GAN-V1 layout assumed by SURVEY.md §0.4; ``HIFIGAN_V2`` / ``HIFIGAN_V3`` are the
other two published layouts.
"""
import copy

_SPEC_MAX = [0.03640973940491676, 0.039425432682037354, 0.29524752497673035, 0.45784831047058105,
             0.48333120346069336, 0.5335848927497864, 0.6071611046791077, 0.5474293828010559,
             0.6076506972312927, 0.5390501022338867, 0.5743886232376099, 0.485751211643219,
             0.4248744249343872, 0.4843744933605194, 0.43331536650657654, 0.5356124639511108,
             0.4875929355621338, 0.48614853620529175, 0.44228559732437134, 0.5027499198913574,
             0.6554337739944458, 0.3469322919845581, 0.33981558680534363, 0.37933868169784546,
             0.34751009941101074, 0.22094282507896423, 0.252963662147522, 0.18274202942848206,
             0.1976650059223175, 0.1770155429840088, 0.18206502497196198, 0.1002601608633995,
             0.18640224635601044, 0.27240633964538574, 0.04153885692358017, -0.010289354249835014,
             -0.012929759919643402, 0.035185474902391434, 0.18124309182167053, -0.14512233436107635,
             -0.1778590828180313, -0.20491982996463776, -0.30119436979293823, -0.1735714226961136,
             -0.1039585992693901, -0.177497997879982, -0.28803232312202454, -0.24049188196659088,
             -0.4682924747467041, -0.5791841745376587, -0.5170156955718994, -0.6380605697631836,
             -0.7147259712219238, -0.6607836484909058, -0.7288452982902527, -0.6338580250740051,
             -0.7092624306678772, -0.8101216554641724, -0.7633087038993835, -0.8251329660415649,
             -0.6936700940132141, -0.5180960297584534, -0.7972619533538818, -0.807314932346344,
             -0.7151175737380981, -0.7785399556159973, -0.8709449768066406, -0.8360402584075928,
             -0.8253681659698486, -0.9778416156768799, -1.12929368019104, -1.3274869918823242,
             -1.3071579933166504, -1.5234452486038208, -1.6191706657409668, -1.708594799041748,
             -1.8246771097183228, -1.9193823337554932, -2.1361801624298096, -2.3829283714294434]

DEFAULT_HPARAMS = {
    "hidden_size": 256, "enc_layers": 4, "dec_layers": 4, "num_heads": 2,
    "enc_ffn_kernel_size": 9, "dec_ffn_kernel_size": 9, "ffn_act": "gelu", "ffn_padding": "SAME",
    "dur_predictor_layers": 2, "dur_predictor_kernel": 3, "predictor_hidden": -1, "predictor_kernel": 5,
    "use_pos_embed": True, "encoder_type": "fft", "decoder_type": "fft", "dur_loss": "mse",
    "use_pitch_embed": True, "use_energy_embed": False, "pitch_type": "frame",
    "mel_vmin": -6, "mel_vmax": 1.5, "timesteps": 100, "K_step": 100, "f0_timesteps": 100,
    "use_spk_id": False, "use_spk_embed": True, "num_spk": 150, "emo": True, "emo_size": 256, "style": True,
    "umln": True, "nRQ": 128, "rq_depth": 4, "f0_gen": "gmdiff", "f0_residual_layers": 10,
    "f0_residual_channels": 192, "f0_dilation_cycle_length": 4, "f0_max_beta": 0.06,
    "decoder": "diffsinger", "residual_layers": 20, "residual_channels": 256,
    "dilation_cycle_length": 4, "max_beta": 0.06, "schedule_type": "linear", "keep_bins": 80,
    "audio_sample_rate": 48000, "hop_size": 256, "audio_num_mel_bins": 80, "max_frames": 3000,
    "vocoder": "HifiGAN_NSF", "use_nsf": True, "pitch_norm": "log", "use_uv": True,
    "diff_decoder_type": "wavenet", "diff_start": 100000, "rq_start": 20500, "forcing": 20000,
    "predictor_grad": 1.0, "use_txt_cond": True, "vocoder_ckpt": "checkpoints/hifigan",
    "vocoder_denoise_c": 0.0, "spec_min": [-6.0] * 80, "spec_max": _SPEC_MAX,
    "processed_data_dir": "data/processed/style", "exp_name": "",
    # not a reference key: precision of the tensor-core GEMMs of the mel DiffNet and the vocoder (TC_PRECISIONS)
    "tc_precision": "split",
    # not a reference key: True admits the two model options of the reference's code that egs/stylesinger.yaml does not
    # select, decoder 'fft' and use_spk_id (EXTENDED_MODELS).  Without it resolve keeps to the yaml's model family
    "extended_models": False,
}

# The reference options that need hparams['extended_models'] = True: the FastSpeech 2 mel decoder alone (decoder 'fft',
# stylesinger.py:185-186) and speaker ids (use_spk_id, fs2.py:37-43).  egs/stylesinger.yaml selects neither; a
# checkpoint trained with one says so in its own hparams, and the caller states that it means to run such a model.
EXTENDED_MODELS = ("decoder: fft", "use_spk_id: True")

# hparams['tc_precision'] -> SSB_TC_SPLIT / SSB_TC_FP16.  'split' (the default): fp32 operands as fp16 hi/lo planes, 3 MMAs
# per K step, mel within 1e-3 of the fp32 reference.  'fp16': one MMA on operands rounded once to fp16 - a third of the
# MMAs, at the accuracy cost README "Single-pass fp16 mode" states.  Applies to the mel DiffNet and the vocoder only.
TC_PRECISIONS = {"split": 0, "fp16": 1}

# HiFi-GAN-V1 style generator; product(upsample_rates) must equal hop_size (256).
DEFAULT_VOCODER_CONFIG = {
    "upsample_rates": [8, 8, 2, 2],
    "upsample_kernel_sizes": [16, 16, 4, 4],
    "upsample_initial_channel": 512,
    "resblock": "1",
    "resblock_kernel_sizes": [3, 7, 11],
    "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]],
    "use_pitch_embed": True,
    "audio_sample_rate": 48000,
    "audio_num_mel_bins": 80,
    "hop_size": 256,
}

# The two other published HiFi-GAN layouts (Kong et al. 2020, config_v2.json / config_v3.json), with the NSF source and
# the rates that give StyleSinger's hop of 256.  V2: V1's layout at 128 initial channels (stages of 64, 32, 16 and 8
# channels).  V3: ResBlock2 (two single convs per block, two dilations each) over three upsampling stages.
HIFIGAN_V2 = dict(DEFAULT_VOCODER_CONFIG, upsample_initial_channel=128)
HIFIGAN_V3 = dict(DEFAULT_VOCODER_CONFIG, upsample_rates=[8, 8, 4], upsample_kernel_sizes=[16, 16, 8],
                  upsample_initial_channel=256, resblock="2", resblock_kernel_sizes=[3, 5, 7],
                  resblock_dilation_sizes=[[1, 2], [2, 6], [3, 12]])

# Boolean model switches (egs/stylesinger.yaml "choices of models", plus use_txt_cond, stylesinger.py:94,317): which
# modules StyleSinger.__init__ builds and which terms its forward adds.  Order = the ssb_model_switches fields.
SWITCHES = ("emo", "style", "umln", "use_txt_cond")


def switches(hp):
    """The model switches of a resolved hparams dict, as {name: bool}."""
    return {k: bool(hp[k]) for k in SWITCHES}


# Mutable module-level dict with the same role as the reference's global `hparams`
# (reference utils/hparams.py:8).
hparams = copy.deepcopy(DEFAULT_HPARAMS)


def resolve(user=None, **overrides):
    """Return a full hparams dict: defaults <- user dict (e.g. the reference's) <- overrides."""
    hp = copy.deepcopy(DEFAULT_HPARAMS)
    if user:
        hp.update({k: v for k, v in user.items()})
    hp.update(overrides)
    _check_supported(hp)
    return hp


def set_hparams(user=None, **overrides):
    hp = resolve(user, **overrides)
    hparams.clear()
    hparams.update(hp)
    return hparams


def _check_supported(hp):
    """The CUDA path implements exactly the configuration egs/stylesinger.yaml selects.
    Anything else fails loudly instead of silently computing something different."""
    prodiff = hp.get("decoder") == "prodiff"  # the ProDiff teacher of the commented block egs/stylesinger.yaml:145-155
    # decoder 'fft': the FastSpeech 2 decoder's mel is the output (stylesinger.py:185-186); no diffusion hparam is read
    fft = hp.get("decoder") == "fft"
    # use_spk_id: spk_embed_proj is an Embedding(num_spk + 1, 256) over speaker ids (fs2.py:37-43), whatever use_spk_embed
    spk_id = hp.get("use_spk_id") is True
    # f0_gen 'conv': two FastSpeech-2 PitchPredictors instead of the two F0 diffusion samplers (stylesinger.py:66-82);
    # f0_timesteps / f0_max_beta are then unread
    conv_f0 = hp.get("f0_gen") == "conv"
    req = {"encoder_type": "fft", "decoder_type": "fft", "ffn_act": "gelu", "ffn_padding": "SAME",
           "dur_loss": "mse", "pitch_type": "frame", "f0_gen": "conv" if conv_f0 else "gmdiff",
           "decoder": "prodiff" if prodiff else "fft" if fft else "diffsinger",
           "diff_decoder_type": "wavenet", "pitch_norm": "log", "use_uv": True,
           "use_spk_id": True if spk_id else False, "use_pitch_embed": True, "use_energy_embed": False,
           "use_pos_embed": True, "num_heads": 2, "hidden_size": 256}
    if not fft:  # the schedule belongs to the mel sampler, which an FFT model does not have
        req["schedule_type"] = "vpsde" if prodiff else "linear"
    if not spk_id:  # with neither option the reference builds no spk_embed_proj, yet its forward calls it
        req["use_spk_embed"] = True
    if (fft or spk_id) and hp.get("extended_models") is not True:
        raise NotImplementedError(
            f"stylesinger_b200: {' and '.join(o for o, on in zip(EXTENDED_MODELS, (fft, spk_id)) if on)} is outside the "
            f"egs/stylesinger.yaml model family; set hparams['extended_models'] = True to run such a checkpoint")
    if not isinstance(hp.get("extended_models"), bool):
        raise NotImplementedError(f"stylesinger_b200: hparams['extended_models'] must be True or False, got "
                                  f"{hp.get('extended_models')!r}")
    if not spk_id and hp.get("use_spk_embed") is False:
        raise NotImplementedError("stylesinger_b200: use_spk_id and use_spk_embed are both False - the reference then builds "
                                  "no spk_embed_proj (fs2.py:37-43), which StyleSinger.forward calls")
    for k, v in req.items():
        if hp.get(k) != v:
            raise NotImplementedError(
                f"stylesinger_b200 implements the egs/stylesinger.yaml configuration only: "
                f"hparams[{k!r}]={hp.get(k)!r}, required {v!r}")
    # the model switches of egs/stylesinger.yaml's "choices of models" block (stylesinger.py:53-64,92-110,131-172,317-326)
    for k in SWITCHES:
        if not isinstance(hp.get(k), bool):
            raise NotImplementedError(f"stylesinger_b200: hparams[{k!r}] must be True or False, got {hp.get(k)!r}")
    if hp.get("rel_pos"):
        raise NotImplementedError("rel_pos is not selected by egs/stylesinger.yaml")
    if hp.get("tc_precision") not in TC_PRECISIONS:
        raise ValueError(f"tc_precision must be one of {sorted(TC_PRECISIONS)}, got {hp.get('tc_precision')!r}")
    if prodiff or fft:  # ProDiffusion.forward(infer=True) never reads K_step or pndm_speedup (prodiff.py:204-222), and an
        return          # FFT model has no diffusion at all
    # shallow diffusion (DiffusionDecoder.forward, shallow_diffusion_tts.py:297-304): q_sample at K_step - 1 of the
    # timesteps-long schedule, then K_step reverse steps; beyond timesteps the reference indexes past its buffers
    K = int(hp["K_step"])
    if not (1 <= K <= int(hp["timesteps"])):
        raise ValueError(f"K_step must be in [1, timesteps = {hp['timesteps']}], got {K}")
    if hp.get("pndm_speedup"):  # PLMS sampler over the mel denoiser (SURVEY.md §8 f2, ssb_mel_diffusion_sample_plms)
        k = int(hp["pndm_speedup"])
        if not (1 <= k < K):
            raise ValueError(f"pndm_speedup must be in [1, K_step = {K}), got {k}")
