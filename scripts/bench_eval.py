"""Evaluation data path, one run of each: the KITTI flow-PNG reader (NumPy vs the GPU decoder), the batch loader's
items/s by worker count, the metrics kernel per batch, and `evaluate` pairs/s next to the model's own rate.

    python scripts/bench_eval.py [--out results/bench_eval.json]

A synthetic tree is written to a temporary directory: Sintel-shaped 436x1024 frames with .flo flows, and KITTI-shaped
375x1242 frames with 16-bit flow PNGs whose rows cycle through all five PNG filter types.  Prints one JSON line per
measurement, starting with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import tf_raft_b200 as T  # noqa: E402
from tf_raft_b200 import datasets as D  # noqa: E402
from tf_raft_b200.datasets import frame_utils  # noqa: E402
from test_gpu_eval import encode_png16  # noqa: E402

RESULTS = []


def emit(**kw):
    RESULTS.append(kw)
    print(json.dumps(kw), flush=True)


def write_tree(root, n_sintel, n_kitti, seed=0):
    rng = np.random.default_rng(seed)

    def frame(h, w):
        base = rng.integers(0, 256, (h // 4 + 1, w // 4 + 1, 3)).astype(np.uint8)
        return (np.kron(base, np.ones((4, 4, 1), np.uint8))[:h, :w] + rng.integers(0, 8, (h, w, 3))).astype(np.uint8)

    d = os.path.join(root, 'sintel', 'training')
    os.makedirs(os.path.join(d, 'clean', 'scene_1'))
    os.makedirs(os.path.join(d, 'flow', 'scene_1'))
    for i in range(n_sintel + 1):
        frame_utils.write_png(os.path.join(d, 'clean', 'scene_1', 'frame_%04d.png' % (i + 1)), frame(436, 1024))
    for i in range(n_sintel):
        frame_utils.write_flow(os.path.join(d, 'flow', 'scene_1', 'frame_%04d.flo' % (i + 1)),
                               rng.normal(0, 10, (436, 1024, 2)).astype(np.float32))
    d = os.path.join(root, 'kitti', 'training')
    os.makedirs(os.path.join(d, 'image_2'))
    os.makedirs(os.path.join(d, 'flow_occ'))
    for i in range(n_kitti):
        for t in (10, 11):
            frame_utils.write_png(os.path.join(d, 'image_2', '%06d_%d.png' % (i, t)), frame(375, 1242))
        rgb = np.empty((375, 1242, 3), np.uint16)
        rgb[..., :2] = np.clip(64 * rng.normal(0, 10, (375, 1242, 2)) + 2 ** 15, 0, 65535)
        rgb[..., 2] = rng.random((375, 1242)) < 0.3
        encode_png16(os.path.join(d, 'flow_occ', '%06d_10.png' % i), rgb, [0, 1, 2, 3, 4])


def cuda_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--pairs', type=int, default=16)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_eval needs a GPU'
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    emit(what='device', card=card)
    with tempfile.TemporaryDirectory() as root:
        write_tree(root, args.pairs, args.pairs)
        kitti, sintel = D.KITTI(root=os.path.join(root, 'kitti')), D.MpiSintel(root=os.path.join(root, 'sintel'))
        paths = kitti.flow_list

        # 1. the KITTI flow reader
        t = time.perf_counter()
        frame_utils.read_flow_kitti(paths[0])
        emit(what='png_numpy_reader', ms_per_file=1e3 * (time.perf_counter() - t), files=1)
        D.read_flow_kitti_batch(paths[:2])
        torch.cuda.synchronize()
        t = time.perf_counter()
        D.read_flow_kitti_batch(paths)
        torch.cuda.synchronize()
        emit(what='png_gpu_read_flow_kitti_batch', ms_per_file=1e3 * (time.perf_counter() - t) / len(paths),
             files=len(paths), note='host inflate + upload + decode')
        from tf_raft_b200.datasets.png16 import decode_png16, pack_rows
        inflated = [frame_utils.inflate_png16(p) for p in paths]
        offsets, _ = pack_rows(inflated)
        data = torch.from_numpy(np.frombuffer(b''.join(r for r, _, _ in inflated), np.uint8).copy()).cuda()
        layout = [(o, h, w) for o, (_, h, w) in zip(offsets, inflated)]
        status = torch.empty(len(paths), dtype=torch.int32, pin_memory=True)
        ms = cuda_ms(lambda: decode_png16(data, layout, paths, status_host=status), 5)
        emit(what='png_gpu_decode_launch', ms_per_batch=ms, ms_per_file=ms / len(paths), files=len(paths))
        ms1 = cuda_ms(lambda: decode_png16(data, layout[:1], paths[:1], status_host=status[:1]), 5)
        emit(what='png_gpu_decode_launch', ms_per_batch=ms1, files=1)

        # 2. the loader, evaluation mode
        for ds, name in ((sintel, 'sintel 436x1024'), (kitti, 'kitti 375x1242')):
            for workers in (1, 2, 4, 8):
                t = time.perf_counter()
                n = sum(len(b[4]) for b in ds.batches(4, workers=workers))
                torch.cuda.synchronize()
                emit(what='loader_items_per_s', dataset=name, workers=workers, items_per_s=n / (time.perf_counter() - t))

        # 3. the metrics kernel
        for B, H, W in ((8, 448, 1024), (8, 1088, 1920)):
            g = torch.randn(B, H, W, 2, device='cuda') * 20
            p = g + torch.randn_like(g)
            v = (torch.rand(B, H, W, device='cuda') < 0.9).float()
            emit(what='metrics_kernel', batch=[B, H, W], ms_per_batch=cuda_ms(lambda: T.flow_metrics(p, g, v), 50))

        # 4. evaluate vs the model at that shape
        model = T.RAFT(seed=0, device='cuda')
        for ds, name, shape in ((sintel, 'sintel', (448, 1024)), (kitti, 'kitti', (376, 1248))):
            bs = 4
            x = torch.rand(bs, *shape, 3, device='cuda') * 255
            ms = cuda_ms(lambda: model([x, x], training=False, last_only=True), 3)
            T.evaluate(model, ds, batch_size=bs)
            torch.cuda.synchronize()
            t = time.perf_counter()
            T.evaluate(model, ds, batch_size=bs)
            dt = time.perf_counter() - t
            emit(what='evaluate_pairs_per_s', dataset=name, padded=list(shape), batch=bs, iters=model.iters_pred,
                 pairs_per_s=len(ds) / dt, model_pairs_per_s=bs / (ms / 1e3))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(RESULTS, f, indent=1)


if __name__ == '__main__':
    main()
