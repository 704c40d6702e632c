"""Multi-GPU plumbing: the path shards over independent utterances (SURVEY.md §8e), one process per GPU.

No collective sits on the data path.  `torch.distributed` (NCCL over NVLink on the GPU box, gloo in the
CPU tests) is used only for the trivial batch scatter (inputs, ~0.4 MB / utterance) and gather (waveforms)
when a single rank owns the request batch, and for the max-over-ranks timing reduction in bench.py.
"""
from typing import List, Optional

import numpy as np
import torch
import torch.distributed as dist

from .engine import PackedBatch, pack_batch
from .sharding import lpt_assign  # noqa: F401  (re-exported)


def empty_batch() -> PackedBatch:
    """The shard of a rank that received no utterance (fewer utterances than ranks)."""
    z = np.zeros(1, np.int32)
    return PackedBatch(0, z, z.copy(), z.copy(), {}, False)


def _p2p_device(device):
    return torch.device(device) if device is not None else torch.device("cpu")


def scatter_utterances(utts: Optional[List[dict]], src: int = 0, device=None, pin: bool = False,
                       keep_on_device: bool = False, emo: bool = True, style: bool = True, spk_id: bool = False):
    """Rank `src` owns `utts` (list of per-utterance CPU tensors, see synth.make_utterance); every rank returns
    (its PackedBatch, the global indices of its utterances).  Metadata goes through scatter_object_list, tensors
    through point-to-point send/recv (NCCL over NVLink when `device` is a CUDA device, gloo on CPU).
    `keep_on_device`: with a CUDA `device` the received shard stays in HBM (no host bounce before the engine call).
    `emo` / `style`: the model switches of the receiving model (pack_batch): without them no emo_embed / reference mels
    are packed or sent.  `spk_id`: the receiving model uses speaker ids (use_spk_id): each shard carries its host ids
    instead of spk_embed rows."""
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = _p2p_device(device)
    if rank == src:
        lens = [int(u["mel2ph"].shape[0]) if "mel2ph" in u else int(len(u["txt_tokens"])) for u in utts]
        bins = lpt_assign(lens, world)
        # fewer utterances than ranks leaves some bins empty: those ranks get an empty batch (B = 0) and skip the compute
        packed = [pack_batch([utts[i] for i in b], use_mel2ph=all("mel2ph" in utts[i] for i in b), emo=emo, style=style,
                             spk_id=spk_id)
                  if b else empty_batch()
                  for b in bins]
        meta = [{"B": p.B, "ph": p.ph_offsets, "ref": p.ref_offsets, "fr": p.frame_offsets, "idx": b, "pad": p.may_have_pad_frames, "spk": p.spk_ids,
                 "shapes": {k: (tuple(v.shape), str(v.dtype)) for k, v in p.t.items()}} for p, b in zip(packed, bins)]
    else:
        packed, meta = None, [None] * world
    mine = [None]
    dist.scatter_object_list(mine, meta if rank == src else None, src=src)
    m = mine[0]
    if rank == src:
        for r in range(world):
            if r == src:
                continue
            for k in sorted(packed[r].t.keys()):
                dist.send(packed[r].t[k].to(dev), dst=r)
        pb = packed[src]
        if keep_on_device and dev.type == "cuda":
            pb = pb.to(dev)
    else:
        t = {}
        for k in sorted(m["shapes"].keys()):
            shape, dt = m["shapes"][k]
            buf = torch.empty(shape, dtype=getattr(torch, dt.replace("torch.", "")), device=dev)
            dist.recv(buf, src=src)
            t[k] = buf if (keep_on_device and dev.type == "cuda") else buf.cpu()
        pb = PackedBatch(m["B"], m["ph"], m["ref"], m["fr"], t, m["pad"], m["spk"])
    if pin and torch.cuda.is_available() and not (keep_on_device and dev.type == "cuda"):
        pb = PackedBatch(pb.B, pb.ph_offsets, pb.ref_offsets, pb.frame_offsets, {k: v.pin_memory() for k, v in pb.t.items()},
                         pb.may_have_pad_frames, pb.spk_ids)
    return pb, m["idx"]


def gather_waveforms(wavs: List[np.ndarray], idx: List[int], n_total: int, dst: int = 0, device=None):
    """Inverse of scatter_utterances for the outputs: rank `dst` returns the list of all waveforms in the
    original utterance order, other ranks return None."""
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = _p2p_device(device)
    metas = [None] * world
    dist.all_gather_object(metas, {"idx": list(idx), "lens": [int(len(w)) for w in wavs]})
    if rank == dst:
        out = [None] * n_total
        for i, w in zip(idx, wavs):
            out[i] = np.asarray(w)
        for r in range(world):
            if r == dst:
                continue
            tot = int(sum(metas[r]["lens"]))
            buf = torch.empty(tot, dtype=torch.float32, device=dev)
            if tot:
                dist.recv(buf, src=r)
            h = buf.cpu().numpy()
            o = 0
            for i, n in zip(metas[r]["idx"], metas[r]["lens"]):
                out[i] = h[o:o + n]
                o += n
        return out
    flat = np.concatenate(wavs) if wavs else np.zeros(0, np.float32)
    if flat.size:
        dist.send(torch.from_numpy(np.ascontiguousarray(flat, dtype=np.float32)).to(dev), dst=dst)
    return None


def gather_waveforms_device(wav: torch.Tensor, frame_offsets, hop: int, idx: List[int], n_total: int, dst: int = 0):
    """Gather for device-resident results: `wav` is this rank's tight waveform tensor [sum_frames * hop] on its GPU
    (utterance j of the shard = global utterance idx[j]); shards travel GPU -> GPU over NCCL and rank `dst` copies them
    to pinned host memory once.  Rank `dst` returns the list of all waveforms (numpy views) in the original utterance
    order, other ranks return None."""
    rank, world = dist.get_rank(), dist.get_world_size()
    fo = np.asarray(frame_offsets, np.int64)
    lens = [int(fo[j + 1] - fo[j]) * hop for j in range(len(idx))]
    metas = [None] * world
    dist.all_gather_object(metas, {"idx": list(idx), "lens": lens})
    if rank != dst:
        if wav.numel():
            dist.send(wav.contiguous(), dst=dst)
        return None
    total = int(sum(sum(m["lens"]) for m in metas))
    host = torch.empty(max(total, 1), dtype=torch.float32).pin_memory() if wav.is_cuda else torch.empty(max(total, 1))
    out, o = [None] * n_total, 0
    for r in range(world):
        tot = int(sum(metas[r]["lens"]))
        if r == dst:
            buf = wav.reshape(-1)
        else:
            buf = torch.empty(tot, dtype=torch.float32, device=wav.device)
            if tot:
                dist.recv(buf, src=r)
        host[o:o + tot].copy_(buf[:tot], non_blocking=True)
        for i, n in zip(metas[r]["idx"], metas[r]["lens"]):
            out[i] = (o, n)
            o += n
    if wav.is_cuda:
        torch.cuda.current_stream(wav.device).synchronize()
    h = host.numpy()
    return [h[a:a + n] for a, n in out]
