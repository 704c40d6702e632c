"""On-disk formats either side of the hot path (SURVEY.md section 8f, row f4): the reference's checkpoints and its
binarised `IndexedDataset`, read without importing the reference.

* checkpoints: ``utils/commons/ckpt_utils.py:7-67`` (``model_ckpt_steps_<N>.ckpt`` in a work dir, newest step wins;
  ``state_dict`` either flat with a ``model.`` prefix or nested under the model name) and the vocoder loader
  ``tasks/tts/vocoder_infer/hifigan_nsf.py:24-60`` (``config.yaml`` + ``state_dict['model_gen']``, or
  ``config.json`` + ``generator_v1`` with the ``'generator'`` key).
* datasets: ``utils/commons/indexed_datasets.py:7-39`` (``<prefix>.idx`` = ``np.save`` of ``{'offsets': [...]}``,
  ``<prefix>.data`` = concatenated pickles) and the item -> model-input conversion of
  ``tasks/StyleSinger/dataset.py:41-66,100-130,153-167`` + ``utils/pitch_utils.py:34-62``.

Everything here is host-side Python; the state dicts go to ``ssb_model_create`` / ``ssb_vocoder_create`` unchanged.
"""
import glob
import json
import os
import pickle
import re
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch


# ------------------------------------------------------------------------------------------------ checkpoints
def list_checkpoints(work_dir: str, steps: Optional[int] = None) -> List[str]:
    """``model_ckpt_steps_*.ckpt`` of a work dir, newest step first (ckpt_utils.py:18-24)."""
    pat = os.path.join(work_dir, f"model_ckpt_steps_{'*' if steps is None else steps}.ckpt")
    found = []
    for p in glob.glob(pat):
        m = re.search(r"steps_(\d+)\.ckpt$", p)
        if m:
            found.append((int(m.group(1)), p))
    return [p for _, p in sorted(found, key=lambda t: -t[0])]


def _select_state_dict(sd_all: dict, model_name: str) -> Dict[str, torch.Tensor]:
    """Key resolution of load_ckpt (ckpt_utils.py:37-51)."""
    if any("." in k for k in sd_all.keys()):  # flat: 'model.encoder...' -> 'encoder...'
        pre = model_name + "."
        return {k[len(pre):]: v for k, v in sd_all.items() if k.startswith(pre)}
    if "." not in model_name:
        if model_name not in sd_all:
            raise KeyError(f"checkpoint has no state dict named '{model_name}' (has: {sorted(sd_all)})")
        return dict(sd_all[model_name])
    base, rest = model_name.split(".", 1)
    pre = rest + "."
    return {k[len(pre):]: v for k, v in sd_all[base].items() if k.startswith(pre)}


def load_state_dict(ckpt_base: str, model_name: str = "model") -> Tuple[Dict[str, torch.Tensor], str]:
    """(state dict with the reference's parameter names, path actually read).  ``ckpt_base`` is a checkpoint file or a
    work dir; a dir without checkpoints raises (the reference asserts, ckpt_utils.py:63-65)."""
    if os.path.isfile(ckpt_base):
        path = ckpt_base
    else:
        paths = list_checkpoints(ckpt_base)
        if not paths:
            raise FileNotFoundError(f"ckpt not found in {ckpt_base}")
        path = paths[0]
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    return _select_state_dict(ckpt["state_dict"], model_name), path


def load_vocoder_checkpoint(base_dir: str) -> Tuple[Dict[str, torch.Tensor], dict, str]:
    """(generator state dict incl. weight_g / weight_v, config dict, path) as HifiGAN.__init__ + load_model find them
    (vocoder_infer/hifigan_nsf.py:24-60): ``config.yaml`` + newest ``model_ckpt_steps_*.ckpt`` ['state_dict']['model_gen'],
    else ``config.json`` + ``generator_v1`` ['generator'] (without ``generator_v1``: the one ``generator_v2`` or
    ``generator_v3`` present)."""
    ycfg, jcfg = os.path.join(base_dir, "config.yaml"), os.path.join(base_dir, "config.json")
    if os.path.exists(ycfg):
        import yaml
        paths = list_checkpoints(base_dir)
        if not paths:
            raise FileNotFoundError(f"no model_ckpt_steps_*.ckpt in {base_dir}")
        with open(ycfg) as f:
            cfg = yaml.safe_load(f) or {}
        ck = torch.load(paths[0], map_location="cpu", weights_only=False)
        return dict(ck["state_dict"]["model_gen"]), cfg, paths[0]
    if os.path.exists(jcfg):
        # the reference reads generator_v1 only; a directory of the official V2 or V3 release holds generator_v2 or
        # generator_v3 instead, and its config.json describes that layout
        path = os.path.join(base_dir, "generator_v1")
        if not os.path.exists(path):
            found = [os.path.join(base_dir, n) for n in ("generator_v2", "generator_v3")
                     if os.path.exists(os.path.join(base_dir, n))]
            if len(found) > 1:
                raise ValueError(f"{base_dir} holds both generator_v2 and generator_v3 and no generator_v1: "
                                 "keep the one its config.json describes")
            if found:
                path = found[0]
        with open(jcfg) as f:
            cfg = json.load(f)
        ck = torch.load(path, map_location="cpu", weights_only=False)
        return dict(ck["generator"]), cfg, path
    raise FileNotFoundError(f"neither config.yaml nor config.json in {base_dir}")


# ------------------------------------------------------------------------------------------------ datasets
class IndexedDatasetReader:
    """Random access to ``<prefix>.idx`` / ``<prefix>.data`` (indexed_datasets.py:7-39)."""

    def __init__(self, prefix: str):
        idx = np.load(f"{prefix}.idx", allow_pickle=True).item()
        self.offsets = [int(o) for o in idx["offsets"]]
        self._f = open(f"{prefix}.data", "rb")

    def __len__(self):
        return len(self.offsets) - 1

    def __getitem__(self, i: int):
        if i < 0 or i >= len(self):
            raise IndexError("index out of range")
        self._f.seek(self.offsets[i])
        return pickle.loads(self._f.read(self.offsets[i + 1] - self.offsets[i]))

    def close(self):
        if self._f:
            self._f.close()
            self._f = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        self.close()


def norm_interp_f0(f0_hz: np.ndarray, pitch_norm: str = "log", use_uv: bool = True, f0_mean: float = 400.0,
                   f0_std: float = 100.0) -> Tuple[np.ndarray, np.ndarray]:
    """utils/pitch_utils.py:34-62: uv = (f0 == 0); f0 -> log2(f0 + 1e-8) (or standardised); unvoiced frames are
    linearly interpolated from their voiced neighbours (all-unvoiced: zeros).  Returns (f0 float32, uv float32)."""
    f0 = np.asarray(f0_hz, dtype=np.float64 if np.asarray(f0_hz).dtype == np.float64 else np.float32).copy()
    uv = f0 == 0
    if pitch_norm == "standard":
        f0 = (f0 - f0_mean) / f0_std
    elif pitch_norm == "log":
        f0 = np.log2(f0 + 1e-8)
    if use_uv:
        f0[uv] = 0
    if uv.sum() == len(f0):
        f0[uv] = 0
    elif uv.sum() > 0:
        f0[uv] = np.interp(np.where(uv)[0], np.where(~uv)[0], f0[~uv])
    return f0.astype(np.float32), uv.astype(np.float32)


def pad_f0_to_mel(f0: np.ndarray, n_mel: int, hop_size: int) -> np.ndarray:
    """The f0 track of the pitch extractor aligned to the mel frames, reference inference/StyleSinger.py:116-137 (the lines after
    the parselmouth call): hop 128 -> pad_size 4, hop 256 -> pad_size 2 (anything else is refused like the reference's
    ``assert False``), 2 * pad_size zero frames in front, zeros behind up to ``n_mel`` frames, |length difference| <= 8 asserted,
    the last value repeated if still short, cut to ``n_mel``."""
    if hop_size == 128:
        pad_size = 4
    elif hop_size == 256:
        pad_size = 2
    else:
        raise AssertionError("hop_size must be 128 or 256 (inference/StyleSinger.py:120-125)")
    f0 = np.asarray(f0)
    lpad = pad_size * 2
    rpad = n_mel - len(f0) - lpad
    f0 = np.pad(f0, [[lpad, rpad]], mode="constant")  # like the reference, a track longer than the mel raises here
    delta_l = n_mel - len(f0)
    assert np.abs(delta_l) <= 8
    if delta_l > 0:
        f0 = np.concatenate([f0, [f0[-1]] * delta_l], 0)
    return f0[:n_mel]


def item_to_utterance(item: dict, hparams: dict, with_mel2ph: bool = True) -> Dict[str, torch.Tensor]:
    """One binarised dataset item -> the utterance dict ``engine.pack_batch`` takes, following the test-time sample
    assembly of tasks/StyleSinger/dataset.py (BaseDataset.__getitem__ :41-66, BaseSingerdataset :100-130,
    StyleSinger_dataset :153-167): the target mel / f0 of the item are the style reference of the utterance
    (tasks/StyleSinger/stylesinger.py:168-197 passes ``ref_mels=sample['mels'], ref_f0=sample['f0']``)."""
    mt = int(hparams.get("max_input_tokens", 2000))
    mult = int(hparams.get("frames_multiple", 1))
    mel = np.asarray(item["mel"], np.float32)[: int(hparams.get("max_frames", 3000))]
    mel = mel[: mel.shape[0] // mult * mult]
    m2p = np.asarray(item["mel2ph"])
    T = min(mel.shape[0], int((m2p > 0).sum()), len(item["f0"]))
    f0, _ = norm_interp_f0(np.asarray(item["f0"])[:T], hparams.get("pitch_norm", "log"), hparams.get("use_uv", True),
                           hparams.get("f0_mean", 400.0), hparams.get("f0_std", 100.0))
    u = {"txt_tokens": torch.as_tensor(np.asarray(item["ph_token"])[:mt]).long(),
         "note": torch.as_tensor(np.asarray(item["ep_pitches"])[:mt]).long(),
         "note_dur": torch.as_tensor(np.asarray(item["ep_notedurs"], np.float32)[:mt]).float(),
         "note_type": torch.as_tensor(np.asarray(item["ep_types"])[:mt]).long(),
         "ref_mels": torch.from_numpy(mel[:T].copy()), "ref_f0": torch.from_numpy(f0)}
    if hparams.get("use_spk_id"):  # the dataset's speaker id (tasks/StyleSinger/dataset.py:63-64,93-95)
        u["spk_id"] = int(item["spk_id"])
    else:
        u["spk_embed"] = torch.as_tensor(np.asarray(item["spk_embed"], np.float32)).float().reshape(-1)
    if hparams.get("emo", True):  # a model without emo reads no emotion embedding (the item may have none)
        u["emo_embed"] = torch.as_tensor(np.asarray(item["emo_embed"], np.float32)).float().reshape(-1)
    if with_mel2ph:
        u["mel2ph"] = torch.as_tensor(m2p[:T]).long()
    u["item_name"] = item.get("item_name")
    return u
