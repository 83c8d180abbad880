"""Training throughput of `RAFT.fit` against a bare loop of `train_step`, at the Chairs config.

    python scripts/bench_fit.py --out DIR [--pairs 40 --epochs 3 --windows 2]

train_chairs.yml's setup: RAFT, batch 4, 368x496 crops (min_scale -0.1, max_scale 1.0, flips), 12 iterations,
AdamW under the cyclical schedule, on a synthetic FlyingChairs tree of `--pairs` 384x512 .ppm / .flo pairs written to a
temporary directory.  Two rates, in pairs/s, alternating in `--windows` windows (median and each window reported):
  * fit: `raft.fit(chairs.batches(4, repeat=True), steps_per_epoch=pairs // 4, epochs=--epochs)` with the reference's
    callbacks (TensorBoard, VisFlowCallback with 4 random pairs at 448x1024, ModelCheckpoint on val_epe), validation
    off -- so the loader's reads, the upload, the augmentor, the step and the end-of-epoch callbacks, timed with a
    host clock around the call, which ends in a device synchronise;
  * bare: the same number of `train_step` calls on batches already augmented and resident on the device.
Also: the host time fit spends inside the loader's next() per window, the loader and augmentor alone (pairs/s, with a synchronise per batch), one VisFlowCallback epoch end and one
`save_weights` with the Adam state (seconds; ModelCheckpoint does not save with validation off, as the reference's
ModelCheckpoint(monitor='val_epe') would not).  The GPU's name, power limit and maximum SM clock are read (nvidia-smi,
query only) in the same run: one JSON line on stdout and in DIR/bench_fit.json.
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import shutil
import tempfile
import time
import warnings

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import tf_raft_b200 as T  # noqa: E402
from tf_raft_b200.datasets import FlyingChairs, frame_utils  # noqa: E402

AUG = {'crop_size': (368, 496), 'min_scale': -0.1, 'max_scale': 1.0, 'do_flip': True}
BATCH, H, W = 4, 384, 512


def gpu_info():
    try:
        res = subprocess.run(['nvidia-smi', f'--id={torch.cuda.current_device()}',
                              '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=60)
        return res.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f'nvidia-smi unavailable: {e}'


def write_tree(root, n, seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    data = os.path.join(root, 'data')
    os.makedirs(data)
    for i in range(n):
        for t in (1, 2):
            base = rng.integers(0, 256, (H // 8, W // 8, 3)).astype(np.uint8)
            Image.fromarray(np.kron(base, np.ones((8, 8, 1), np.uint8))).save(os.path.join(data, f'{i + 1:05d}_img{t}.ppm'))
        frame_utils.write_flow(os.path.join(data, f'{i + 1:05d}_flow.flo'), rng.normal(0, 5, (H, W, 2)).astype(np.float32))
    split = os.path.join(root, 'split.txt')
    np.savetxt(split, np.ones(n, np.int32), fmt='%d')
    return data, split


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--pairs', type=int, default=40)
    ap.add_argument('--epochs', type=int, default=3)
    ap.add_argument('--windows', type=int, default=2)
    ap.add_argument('--workers', type=int, default=4)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    np.random.seed(0)
    random.seed(0)
    tmp = tempfile.mkdtemp(prefix='bench_fit_')
    data, split = write_tree(tmp, args.pairs)
    chairs = FlyingChairs(AUG, split='training', split_txt=split, root=data)
    chairs.shuffle()
    vis = FlyingChairs(split='training', split_txt=split, root=data)
    steps = args.pairs // BATCH
    raft = T.RAFT(drop_rate=0, iters=12, iters_pred=24)
    sched = T.CyclicalLearningRate(4e-4, 8e-4, 1000, T.first_cycle_scaler, 'cycle')
    raft.compile(optimizer=T.AdamW(weight_decay=1e-4, learning_rate=sched), clip_norm=1.0)
    logdir = os.path.join(tmp, 'logs')
    vis_cb = T.VisFlowCallback(vis, num_visualize=4, choose_random=True, logdir=os.path.join(logdir, 'predicted_flows'))
    callbacks = [T.TensorBoard(log_dir=os.path.join(logdir, 'history')), vis_cb,
                 T.ModelCheckpoint(os.path.join(logdir, 'checkpoints', 'model'), save_weights_only=True,
                                   monitor='val_epe', mode='min', save_best_only=True)]
    warnings.simplefilter('ignore')                        # ModelCheckpoint's "val_epe not available" each epoch

    stream = chairs.batches(BATCH, workers=args.workers, repeat=True)
    resident = [tuple(t.clone() for t in next(stream)) for _ in range(steps)]

    waits = []

    class Timed:
        """The loader as fit sees it, with the host time spent waiting in next() added to waits[-1]."""

        def __init__(self, it):
            self.it = it

        def __iter__(self):
            return self

        def __next__(self):
            t0 = time.perf_counter()
            batch = next(self.it)
            waits[-1] += time.perf_counter() - t0
            return batch

    def run_fit(epochs):
        waits.append(0.0)
        raft.fit(Timed(chairs.batches(BATCH, workers=args.workers, repeat=True)), epochs=epochs, steps_per_epoch=steps,
                 callbacks=callbacks, verbose=0)

    def run_bare(epochs):
        for _ in range(epochs):
            raft.reset_metrics()
            for batch in resident:
                raft.train_step(batch)

    timed(lambda: run_fit(1))                              # warm-up: allocations, module loads, the 448x1024 forward
    timed(lambda: run_bare(1))
    n_pairs = args.epochs * steps * BATCH
    fit_rates, bare_rates = [], []
    for _ in range(args.windows):
        bare_rates.append(n_pairs / timed(lambda: run_bare(args.epochs)))
        fit_rates.append(n_pairs / timed(lambda: run_fit(args.epochs)))

    def run_loader():
        for _ in range(args.epochs * steps):
            next(stream)
            torch.cuda.synchronize()
    loader_rate = n_pairs / timed(run_loader)
    vis_s = timed(lambda: vis_cb.on_epoch_end(0))
    save_s = timed(lambda: raft.save_weights(os.path.join(tmp, 'save', 'model')))
    fit_pps, bare_pps = statistics.median(fit_rates), statistics.median(bare_rates)
    result = {'bench': 'fit', 'config': 'chairs: RAFT, batch 4, 368x496 crops of 384x512, 12 iterations',
              'steps_per_epoch': steps, 'epochs': args.epochs, 'fit_pairs_per_s': round(fit_pps, 3),
              'bare_pairs_per_s': round(bare_pps, 3), 'fit_vs_bare': round(fit_pps / bare_pps - 1, 4),
              'fit_windows': [round(r, 3) for r in fit_rates], 'bare_windows': [round(r, 3) for r in bare_rates],
              'fit_loader_wait_s': [round(w, 3) for w in waits[1:]], 'loader_pairs_per_s': round(loader_rate, 2),
              'vis_callback_s': round(vis_s, 3),
              'save_weights_s': round(save_s, 3), 'gpu': gpu_info()}
    line = json.dumps(result)
    print(line)
    with open(os.path.join(args.out, 'bench_fit.json'), 'w') as f:
        f.write(line + '\n')
    shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    main()
