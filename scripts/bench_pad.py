"""RAFT's evaluation protocol, one run: the pad kernel per batch, `evaluate` with zero against replicate padding, and
warm-started sequence evaluation against pairwise evaluation.

    python scripts/bench_pad.py [--out results/bench_pad.json] [--rounds 3]

A synthetic tree is written to a temporary directory from a seed: Sintel-shaped 436x1024 scenes with .flo flows and
KITTI-shaped 375x1242 pairs with flow PNGs.  The compared `evaluate` configurations run alternately, `--rounds` times
each, after one warm-up of each; the median and the range are reported.  Prints one JSON line per measurement,
starting with the card's name and power limit.
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

import tf_raft_b200 as T  # noqa: E402
from tf_raft_b200 import _lib  # noqa: E402
from tf_raft_b200 import datasets as D  # noqa: E402
from tf_raft_b200.datasets import frame_utils  # noqa: E402
from tf_raft_b200.preprocess import _DTYPES, REPLICATE, ZERO, _PadPlane, pad_planes, placement  # noqa: E402

RESULTS = []


def emit(**kw):
    RESULTS.append(kw)
    print(json.dumps(kw), flush=True)


def write_tree(root, scenes, frames_per_scene, n_kitti, seed=0):
    rng = np.random.default_rng(seed)

    def frame(h, w):
        base = rng.integers(0, 256, (h // 4 + 1, w // 4 + 1, 3)).astype(np.uint8)
        return (np.kron(base, np.ones((4, 4, 1), np.uint8))[:h, :w] + rng.integers(0, 8, (h, w, 3))).astype(np.uint8)

    d = os.path.join(root, 'sintel', 'training')
    for s in range(scenes):
        os.makedirs(os.path.join(d, 'clean', 'scene_%d' % s))
        os.makedirs(os.path.join(d, 'flow', 'scene_%d' % s))
        for i in range(frames_per_scene):
            frame_utils.write_png(os.path.join(d, 'clean', 'scene_%d' % s, 'frame_%04d.png' % (i + 1)), frame(436, 1024))
        for i in range(frames_per_scene - 1):
            frame_utils.write_flow(os.path.join(d, 'flow', 'scene_%d' % s, 'frame_%04d.flo' % (i + 1)),
                                   rng.normal(0, 10, (436, 1024, 2)).astype(np.float32))
    d = os.path.join(root, 'kitti', 'training')
    os.makedirs(os.path.join(d, 'image_2'))
    os.makedirs(os.path.join(d, 'flow_occ'))
    for i in range(n_kitti):
        for t in (10, 11):
            frame_utils.write_png(os.path.join(d, 'image_2', '%06d_%d.png' % (i, t)), frame(375, 1242))
        frame_utils.write_flow_kitti(os.path.join(d, 'flow_occ', '%06d_10.png' % i),
                                     rng.normal(0, 10, (375, 1242, 2)).astype(np.float32),
                                     rng.random((375, 1242)) < 0.3)


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


def pad_jobs(B, h, w, mode):
    """One evaluation batch as the loader pads it: frames replicated, flow and valid zero-filled."""
    H, W = -(-h // 8) * 8, -(-w // 8) * 8
    top, left = placement(h, w, H, W, mode)
    jobs = []
    for _ in range(B):
        for c, dt, fill in ((3, torch.uint8, REPLICATE), (3, torch.uint8, REPLICATE), (2, torch.float32, ZERO),
                            (None, torch.float32, ZERO)):
            shape = (h, w) if c is None else (h, w, c)
            src = torch.randint(0, 255, shape, device='cuda').to(dt)
            dst = torch.empty((H, W) + shape[2:], dtype=dt, device='cuda')
            jobs.append((src, dst, top, left, fill))
    nbytes = sum(s.numel() * s.element_size() + d.numel() * d.element_size() for s, d, *_ in jobs)
    return jobs, nbytes


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--scenes', type=int, default=2)
    ap.add_argument('--frames', type=int, default=9, help='frames per Sintel scene')
    ap.add_argument('--kitti', type=int, default=16)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_pad needs a GPU'
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    emit(what='device', card=card)

    # 1. the pad kernel: one batch's 4B planes, with and without the descriptor upload of each call
    for B, h, w, mode in ((4, 436, 1024, 'sintel'), (8, 375, 1242, 'kitti')):
        jobs, nbytes = pad_jobs(B, h, w, mode)
        call = cuda_ms(lambda: pad_planes(jobs), 50)
        arr = (_PadPlane * len(jobs))()                         # the same descriptors, uploaded once
        for p, (src, dst, top, left, fill) in zip(arr, jobs):
            c = src.shape[2] if src.dim() == 3 else 1
            p.src, p.dst, p.h, p.w, p.c, p.H, p.W = src.data_ptr(), dst.data_ptr(), h, w, c, dst.shape[0], dst.shape[1]
            p.top, p.left, p.dtype, p.mode = top, left, _DTYPES[src.dtype], fill
        dev = torch.frombuffer(bytearray(arr), dtype=torch.uint8).cuda()
        lib = _lib.lib()
        kernel = cuda_ms(lambda: lib.raft_b200_pad_batch(arr, _lib.ptr(dev), len(jobs), _lib.stream()), 200)
        emit(what='pad_kernel', batch=[B, h, w], mode=mode, planes=len(jobs), ms_per_batch_kernel=kernel,
             ms_per_batch_call=call, gb_per_s_kernel=nbytes / kernel / 1e6, bytes_moved=nbytes)

    with tempfile.TemporaryDirectory() as root:
        write_tree(root, args.scenes, args.frames, args.kitti)
        sintel, kitti = D.MpiSintel(root=os.path.join(root, 'sintel')), D.KITTI(root=os.path.join(root, 'kitti'))
        model = T.RAFT(seed=0, device='cuda')

        def compare(name, configs):
            for _, fn in configs:                               # warm-up of every configuration
                timed(fn)
            rates = {k: [] for k, _ in configs}
            for _ in range(args.rounds):
                for k, fn in configs:
                    dt, n = timed(fn)
                    rates[k].append(n / dt)
            for k, r in rates.items():
                emit(what=name, config=k, iters=model.iters_pred, pairs_per_s_median=float(np.median(r)),
                     pairs_per_s_min=min(r), pairs_per_s_max=max(r), rounds=args.rounds)

        def ev(ds, **kw):
            return lambda: (T.evaluate(model, ds, **kw), len(ds))[1]

        # 2. evaluate with zero against replicate padding, alternating
        for ds, name, mode in ((sintel, 'sintel 436x1024', 'sintel'), (kitti, 'kitti 375x1242', 'kitti')):
            compare(f'evaluate {name}', [('zero batch 4', ev(ds, batch_size=4)),
                                         ('replicate batch 4', ev(ds, batch_size=4, padding='replicate',
                                                                  pad_mode=mode))])
        # 3. warm-started sequences against pairs, on the same scenes
        compare('evaluate sintel scenes', [
            ('pairs replicate batch 1', ev(sintel, padding='replicate')),
            ('warm start replicate', ev(sintel, padding='replicate', warm_start=True)),
            ('pairs replicate batch 4', ev(sintel, batch_size=4, padding='replicate'))])
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(RESULTS, f, indent=1)


if __name__ == '__main__':
    main()
