"""Batch test path over the reference's on-disk formats (SURVEY.md section 8f, f4): reads a released acoustic checkpoint
directory, a HiFi-GAN vocoder directory and a binarised IndexedDataset, runs ph -> mel -> wav on the CUDA engine in
ragged batches and writes one wav per item.  Equivalent of `python tasks/run.py --config ... --infer` of the reference
(tasks/StyleSinger/stylesinger.py:168-275, which asserts B=1).

    python tools/infer_dataset.py --ckpt checkpoints/StyleSinger --vocoder checkpoints/hifigan --data data/binary/x/test \
        --out infer_out [--batch 64] [--T 100] [--k-step 50] [--limit N] [--use-gt-dur] [--vocoder-denoise-c 0.1] \
        [--seed S] [--seed-per-item]

Like the reference's test_step (tasks/StyleSinger/stylesinger.py:177-180 with `use_gt_dur: false` in egs/stylesinger.yaml) the
durations come from the duration predictor unless --use-gt-dur is given (then the items' ground-truth mel2ph is fed).

By default each batch draws its noise from one seed (--seed plus the batch's start), so an item's audio depends on
--batch, --limit and the dataset's size.  --seed-per-item gives item i (its index in the dataset) the seed --seed + i:
its wav is then that of StyleSingerInfer.forward_model(item, seed=--seed + i), whatever the batching.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def item_seeds(seed, idx):
    """--seed-per-item: the per-utterance seeds of the dataset items `idx`."""
    return [seed + i for i in idx]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ckpt", required=True, help="work dir with model_ckpt_steps_*.ckpt, or one checkpoint file")
    ap.add_argument("--vocoder", required=True, help="dir with config.yaml + model_ckpt_steps_*.ckpt (or config.json + generator_v1)")
    ap.add_argument("--data", required=True, help="IndexedDataset prefix (<prefix>.idx / <prefix>.data)")
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--T", type=int, default=100)
    ap.add_argument("--k-step", type=int, default=None,
                    help="reference hparam K_step (shallow diffusion): mel reverse steps from q_sample at K-1; default --T")
    ap.add_argument("--limit", type=int, default=0)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--seed-per-item", action="store_true",
                    help="seed item i with --seed + i, so that its audio does not depend on the batching")
    ap.add_argument("--use-gt-dur", action="store_true", help="feed the items' ground-truth mel2ph (reference hparam use_gt_dur)")
    ap.add_argument("--vocoder-denoise-c", type=float, default=0.0,
                    help="reference hparam vocoder_denoise_c: > 0 denoises every waveform (hifigan_nsf.py:14-22,73-74)")
    ap.add_argument("--tc-precision", choices=("split", "fp16"), default="split",
                    help="tensor-core GEMMs of the mel denoiser and the vocoder: 'split' (3 MMAs, the default) or 'fp16' "
                         "(single pass: faster, less accurate; README 'Single-pass fp16 mode')")
    for sw in ("emo", "style", "umln", "use_txt_cond"):  # the checkpoint's model switches (egs/stylesinger.yaml)
        ap.add_argument(f"--{sw.replace('_', '-')}", type=int, choices=(0, 1), default=1,
                        help=f"reference hparam {sw} of the checkpoint (default 1)")
    ap.add_argument("--decoder", choices=("diffsinger", "fft"), default="diffsinger",
                    help="reference hparam decoder of the checkpoint: 'fft' is the FastSpeech 2 decoder alone (no diffusion)")
    ap.add_argument("--use-spk-id", type=int, choices=(0, 1), default=0,
                    help="reference hparam use_spk_id: the checkpoint looks speakers up by the items' spk_id")
    ap.add_argument("--num-spk", type=int, default=150, help="reference hparam num_spk (the speaker table has num_spk + 1 rows)")
    args = ap.parse_args()

    from scipy.io import wavfile
    from stylesinger_b200 import formats
    from stylesinger_b200.hparams import resolve
    from stylesinger_b200.infer import StyleSingerInfer

    hp = resolve(timesteps=args.T, K_step=args.T if args.k_step is None else args.k_step, f0_timesteps=args.T,
                 vocoder_denoise_c=args.vocoder_denoise_c, emo=bool(args.emo), style=bool(args.style),
                 umln=bool(args.umln), use_txt_cond=bool(args.use_txt_cond), tc_precision=args.tc_precision,
                 decoder=args.decoder, use_spk_id=bool(args.use_spk_id), num_spk=args.num_spk,
                 extended_models=args.decoder == "fft" or bool(args.use_spk_id))
    sd, path = formats.load_state_dict(args.ckpt, "model")
    vsd, vcfg, vpath = formats.load_vocoder_checkpoint(args.vocoder)
    print(f"| acoustic checkpoint {path} ({len(sd)} tensors); vocoder {vpath}")
    eng = StyleSingerInfer(hp, None, sd, vsd, vcfg)
    os.makedirs(args.out, exist_ok=True)
    sr = int(hp.get("audio_sample_rate", 48000))
    with formats.IndexedDatasetReader(args.data) as ds:
        n = len(ds) if args.limit <= 0 else min(args.limit, len(ds))
        # length-sorted batches: similar lengths share a batch (the engine is ragged, this only balances tile counts)
        order = sorted(range(n), key=lambda i: len(ds[i]["mel"]))
        for b0 in range(0, n, args.batch):
            idx = order[b0:b0 + args.batch]
            utts = [formats.item_to_utterance(ds[i], hp, with_mel2ph=args.use_gt_dur) for i in idx]
            if args.seed_per_item:
                wavs = eng.infer_batch(utts, seeds=item_seeds(args.seed, idx), use_mel2ph=args.use_gt_dur)
            else:
                wavs = eng.infer_batch(utts, seed=args.seed + b0, use_mel2ph=args.use_gt_dur)
            for i, u, w in zip(idx, utts, wavs):
                name = str(u.get("item_name") or f"item{i}")
                wavfile.write(os.path.join(args.out, name + ".wav"), sr, np.asarray(w, np.float32))
            print(f"| {min(b0 + args.batch, n)}/{n} items", flush=True)


if __name__ == "__main__":
    main()
