"""Cost of conventions='pytorch' (the original RAFT's arithmetic) against the default 'tf-raft', on one GPU.

  * lookup: CUDA-event microseconds per raft_b200_corr_lookup_ex call, sampler 'tf-raft' vs 'grid_sample', the fp32
    output of a 4-level radius-4 pyramid at the benchmark shape (B = 4, 448x512 -> 56x64) and the Chairs shape
    (B = 4, 368x496 -> 46x62), the samplers alternating;
  * model: pairs/s of RAFT inference (f16x2, CUDA graph, last_only) at 448x512 x 12 iterations (batch 4) and
    440x1024 x 32 iterations (batch 1), the two conventions alternating, medians of rounds.
Prints one JSON line with the card's name and power limit; --out DIR also writes it there."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), '..')))


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return torch.cuda.get_device_name()


def lookup_us(T, b, h, w, reps, rounds):
    from tf_raft_b200 import _lib
    g = torch.Generator(device='cuda').manual_seed(0)
    f1 = torch.randn(b, h, w, 256, device='cuda', generator=g)
    f2 = torch.randn(b, h, w, 256, device='cuda', generator=g)
    blocks = {s: T.CorrBlock(f1, f2, 4, 4, sampler=s) for s in ('tf-raft', 'grid_sample')}
    yy, xx = torch.meshgrid(torch.arange(h, device='cuda'), torch.arange(w, device='cuda'), indexing='ij')
    coords = (torch.stack([xx, yy], -1).float()[None].repeat(b, 1, 1, 1)
              + torch.empty(b, h, w, 2, device='cuda').uniform_(-6, 6, generator=g)).contiguous()
    out = torch.empty(b, h, w, 324, device='cuda')
    res = {s: [] for s in blocks}
    for _ in range(rounds):
        for s, cb in blocks.items():
            args = (_lib.ptr_array(cb.corr_pyramid), _lib.ptr(coords), b, h, w, 4, 4, _lib.ptr(out), 324, _lib.SAMPLERS[s])
            for _ in range(5):
                _lib.call('corr_lookup_ex', coords.device, *args)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                _lib.call('corr_lookup_ex', coords.device, *args)
            e1.record()
            e1.synchronize()
            res[s].append(e0.elapsed_time(e1) * 1e3 / reps)
    return {s: float(np.median(v)) for s, v in res.items()}


def pairs_per_s(T, b, H, W, iters, steps, rounds):
    rng = np.random.default_rng(0)
    im1 = torch.from_numpy(rng.uniform(0, 255, (b, H, W, 3)).astype(np.float32)).cuda()
    im2 = torch.roll(im1, 4, dims=2).contiguous()
    models = {c: T.RAFT(conventions=c, precision='f16x2', iters_pred=iters, use_graph=True, device='cuda', seed=1)
              for c in ('tf-raft', 'pytorch')}
    res = {c: [] for c in models}
    for m in models.values():
        for _ in range(3):
            m([im1, im2], training=False, last_only=True)
    for _ in range(rounds):
        for c, m in models.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(steps):
                m([im1, im2], training=False, last_only=True)
            torch.cuda.synchronize()
            res[c].append(b * steps / (time.perf_counter() - t))
    return {c: float(np.median(v)) for c, v in res.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import tf_raft_b200 as T
    torch.backends.cudnn.benchmark = False
    result = {'card': card(),
              'lookup_us': {'bench_4x56x64': lookup_us(T, 4, 56, 64, 200, a.rounds),
                            'chairs_4x46x62': lookup_us(T, 4, 46, 62, 200, a.rounds)},
              'pairs_per_s': {'448x512_b4_12it': pairs_per_s(T, 4, 448, 512, 12, a.steps, a.rounds),
                              '440x1024_b1_32it': pairs_per_s(T, 1, 440, 1024, 32, a.steps, a.rounds)}}
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'bench_pytorch_conventions.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
