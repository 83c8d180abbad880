"""Colour-jitter throughput: FlowAugmentor / SparseFlowAugmentor(colour='torchvision') `.batch` at batch 8, against the
original RAFT's augmentor on the host (torchvision ColorJitter on PIL images, cv2 resize), one sample at a time.

    python scripts/bench_colour_jitter.py --out DIR [--batch 8 --windows 5 --calls 20 --host-samples 8]

Three workloads, seeded synthetic uint8 frames and float32 flows already on the GPU, at RAFT's stage settings:
  * chairs: FlowAugmentor((368, 496)) on 384x512 sources;
  * sintel: FlowAugmentor((368, 768)) on 436x1024 sources;
  * kitti:  SparseFlowAugmentor((288, 960)) on 375x1242 sources with a 25 % valid mask.
For each: samples/s of `.batch(samples)` with fresh parameters from the seeded sampler every call (host draws, upload
and kernels), for colour='torchvision' and, for scale, the default colour='albumentations', from CUDA events around
device-synchronised windows of `--calls` calls after a warm-up, median and best of `--windows`; the device time per
batch of the colour_jitter_* and augment_* kernels from torch.profiler (CUDA activities, a separate run); and
samples/s of oracle/raft_augment.py on the host (needs torchvision, Pillow and OpenCV).  The GPU's name, power limit
and maximum SM clock are read (nvidia-smi, query only) in the same run: one JSON line on stdout and in
DIR/bench_colour_jitter.json.
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

from oracle import raft_augment as R  # noqa: E402
from tf_raft_b200.datasets import FlowAugmentor, SparseFlowAugmentor  # noqa: E402

WORKLOADS = {'chairs': (FlowAugmentor, R.FlowAugmentor, (384, 512), dict(crop_size=(368, 496), min_scale=-0.1,
                                                                         max_scale=1.0, do_flip=True)),
             'sintel': (FlowAugmentor, R.FlowAugmentor, (436, 1024), dict(crop_size=(368, 768), min_scale=-0.2,
                                                                          max_scale=0.6, do_flip=True)),
             'kitti': (SparseFlowAugmentor, R.SparseFlowAugmentor, (375, 1242), dict(crop_size=(288, 960),
                                                                                    min_scale=-0.2, max_scale=0.4,
                                                                                    do_flip=False))}


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


def time_batches(aug, dev, args):
    np.random.seed(1)
    random.seed(2)
    torch.manual_seed(3)
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
    return {'samples_per_s_median': round(statistics.median(rates), 1), 'samples_per_s_best': round(max(rates), 1),
            'window_ms': [round(x, 2) for x in windows]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--windows', type=int, default=5)
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--host-samples', type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_colour_jitter.py needs a CUDA device')
    os.makedirs(args.out, exist_ok=True)
    result = {'metric': 'augmented samples/s (.batch, batch %d)' % args.batch, 'gpu': gpu_info(),
              'device': torch.cuda.get_device_name(), 'batch': args.batch, 'workloads': {}}
    rng = np.random.default_rng(0)
    for name, (cls, ref_cls, (h, w), aug_args) in WORKLOADS.items():
        sparse = cls is SparseFlowAugmentor
        host = make_samples(args.batch, h, w, sparse, rng)
        dev = [tuple(torch.from_numpy(a).cuda() for a in s) for s in host]
        aug = cls(colour='torchvision', **aug_args)
        entry = {'source': [h, w], 'crop': list(aug_args['crop_size']),
                 'torchvision': time_batches(aug, dev, args),
                 'albumentations': time_batches(cls(**aug_args), dev, args)}
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                aug.batch(dev)
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            if 'colour_jitter_' in e.key or 'augment_' in e.key:
                kernels[e.key.split('(')[0].replace('void ', '').replace('raft::', '')] = \
                    round(e.device_time_total / 1e3 / args.calls, 4)
        entry['kernel_ms_per_batch'] = kernels
        entry['colour_jitter_kernel_ms_per_batch'] = round(sum(v for k, v in kernels.items() if 'colour_jitter' in k), 4)
        ref = ref_cls(**aug_args)
        np.random.seed(4)
        torch.manual_seed(5)
        n = args.host_samples
        t = time.perf_counter()
        for i in range(n):
            ref(*[a.copy() for a in host[i % len(host)]])
        entry['host_torchvision_pil_samples_per_s'] = round(n / (time.perf_counter() - t), 1)
        result['workloads'][name] = entry
    line = json.dumps(result)
    print(line)
    with open(os.path.join(args.out, 'bench_colour_jitter.json'), 'w') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
