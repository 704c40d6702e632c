"""SURVEY.md section 8e on hardware: NCCL scatter of the ragged inputs + per-rank compute + NCCL gather of the waveforms
(world size 2, one process per GPU).  Needs >= 2 GPUs; skipped on a single-GPU box."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dev = torch.device(f"cuda:{rank}")
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from stylesinger_b200 import synth
        from stylesinger_b200.dist import gather_waveforms_device, scatter_utterances
        from stylesinger_b200.engine import pack_batch
        from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG, resolve
        from stylesinger_b200.infer import StyleSingerInfer
        from stylesinger_b200.sharding import lpt_assign
        T, n = 4, 6
        hp = resolve(timesteps=T, K_step=T, f0_timesteps=T)
        eng = StyleSingerInfer(hp, dev, synth.acoustic_state_dict(hp, seed=0), synth.vocoder_state_dict(DEFAULT_VOCODER_CONFIG, seed=0),
                               DEFAULT_VOCODER_CONFIG)
        mk = lambda i: synth.make_utterance(0.4 + 0.25 * i, utt_idx=i, ref_frames=40 + 3 * i)
        utts = [mk(i) for i in range(n)] if rank == 0 else None
        pb, idx = scatter_utterances(utts, src=0, device=dev, keep_on_device=True)
        assert all(v.is_cuda for v in pb.t.values())
        _, _, wav, fo = eng.run_device(pb, seed=5)
        out = gather_waveforms_device(wav, fo, eng.vocoder.hop, idx, n, dst=0)
        ok, detail = True, ""
        if rank == 0:
            lens = [int(u["mel2ph"].shape[0]) for u in utts]
            bins = lpt_assign(lens, world)
            for b in bins:  # same shard composition + same seed => the same Philox streams => bit-identical waveforms
                pbl = pack_batch([utts[i] for i in b]).to(dev)
                _, _, w, fol = eng.run_device(pbl, seed=5)
                w = w.cpu().numpy()
                for j, i in enumerate(b):
                    ref = w[int(fol[j]) * 256:int(fol[j + 1]) * 256]
                    if out[i] is None or not np.array_equal(out[i], ref):
                        ok, detail = False, f"utterance {i} differs"
            ok = ok and all(len(out[i]) == lens[i] * 256 for i in range(n))
        q.put((rank, ok, detail, sorted(idx)))
    finally:
        dist.destroy_process_group()


def test_scatter_compute_gather_over_nccl_world2():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in range(2)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert all(r[1] for r in res), res
    assert sorted(sum((r[3] for r in res), [])) == list(range(6))
