"""Training-augmentation throughput: FlowAugmentor / SparseFlowAugmentor `.batch` at batch 8.

    python scripts/bench_augment.py --out DIR [--batch 8 --windows 5 --calls 20]

Three workloads, seeded synthetic uint8 frames and float32 flows already on the GPU:
  * chairs: FlowAugmentor((368, 496)) on 384x512 sources;
  * sintel: FlowAugmentor((368, 768)) on 436x1024 sources;
  * kitti:  SparseFlowAugmentor((288, 960)) on 375x1242 sources with a 25 % valid mask.
For each: samples/s of `.batch(samples)` with fresh parameters from the seeded sampler every call (the host draws, the
parameter upload and the kernels), from CUDA events around device-synchronised windows of `--calls` calls after a
warm-up, median and best of `--windows`; the device time of the augment_* kernels per batch from torch.profiler (CUDA
activities, a separate run); and the host time per sample of the NumPy restatement (oracle/augment_np.py) for scale.
The GPU's name, power limit and maximum SM clock are read (nvidia-smi, query only) in the same run: one JSON line on
stdout and in DIR/bench_augment.json.
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import augment_np as A  # noqa: E402
from tf_raft_b200.datasets import FlowAugmentor, SparseFlowAugmentor  # noqa: E402

WORKLOADS = {'chairs': (FlowAugmentor, (368, 496), (384, 512)),
             'sintel': (FlowAugmentor, (368, 768), (436, 1024)),
             'kitti': (SparseFlowAugmentor, (288, 960), (375, 1242))}


def gpu_info():
    try:
        res = subprocess.run(['nvidia-smi', f'--id={torch.cuda.current_device()}',
                              '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=60)
        return res.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f'nvidia-smi unavailable: {e}'


def make_samples(n, h, w, sparse, rng):
    out = []
    for _ in range(n):
        s = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8), rng.integers(0, 256, (h, w, 3), dtype=np.uint8),
             (rng.standard_normal((h, w, 2)) * 20).astype(np.float32)]
        if sparse:
            s.append((rng.uniform(size=(h, w)) < 0.25).astype(np.float32))
        out.append(s)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--windows', type=int, default=5)
    ap.add_argument('--calls', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_augment.py needs a CUDA device')
    os.makedirs(args.out, exist_ok=True)
    result = {'metric': 'augmented samples/s (.batch, batch %d)' % args.batch, 'gpu': gpu_info(),
              'device': torch.cuda.get_device_name(), 'batch': args.batch, 'workloads': {}}
    rng = np.random.default_rng(0)
    for name, (cls, crop, (h, w)) in WORKLOADS.items():
        sparse = cls is SparseFlowAugmentor
        aug = cls(crop)
        host = make_samples(args.batch, h, w, sparse, rng)
        dev = [tuple(torch.from_numpy(a).cuda() for a in s) for s in host]
        np.random.seed(1)
        random.seed(2)
        for _ in range(3):
            aug.batch(dev)
        windows = []
        for _ in range(args.windows):
            torch.cuda.synchronize()
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(args.calls):
                aug.batch(dev)
            end.record()
            torch.cuda.synchronize()
            windows.append(start.elapsed_time(end))
        rates = [args.batch * args.calls / (ms / 1e3) for ms in windows]
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                aug.batch(dev)
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            if 'augment_' in e.key:
                kernels[e.key.split('(')[0].replace('void ', '').replace('raft::', '')] = \
                    round(e.device_time_total / 1e3 / args.calls, 4)
        params = [aug.sample_params(h, w) for _ in range(3)]
        t = time.perf_counter()
        for s, p in zip(host, params):
            (A.augment_sparse if sparse else A.augment_dense)(*s, p)
        oracle_ms = (time.perf_counter() - t) * 1e3 / len(params)
        result['workloads'][name] = {
            'source': [h, w], 'crop': list(crop), 'samples_per_s_median': round(statistics.median(rates), 1),
            'samples_per_s_best': round(max(rates), 1), 'window_ms': [round(x, 2) for x in windows],
            'kernel_ms_per_batch': kernels, 'kernel_ms_per_batch_total': round(sum(kernels.values()), 4),
            'oracle_host_ms_per_sample': round(oracle_ms, 1)}
    line = json.dumps(result)
    print(line)
    with open(os.path.join(args.out, 'bench_augment.json'), 'w') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
