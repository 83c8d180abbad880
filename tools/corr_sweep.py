"""SURVEY.md section 8(d), config 5: correlation-pyramid build (K1) and lookup (K2) over feature-map sizes.

For every g in {32, 48, 64, 96, 128, 192, 256}: fmap1, fmap2 ~ N(0, 1) fp32 (1, g, g, 256), 4 levels, radius 4;
lookup coordinates = grid + U(-8, 8)^2 (seed 2) and the integer grid (the iteration-0 case, where every level-0 tap is
exactly 0).  Prints CUDA-event times and the achieved algorithmic bandwidth (section 8(d) byte counts):
  K1: write 4 * sum_l N * N_l  +  read 2 * N * C * 4        K2: 2904 B per query (read 1600, coords 8, write 1296)
usage: python tools/corr_sweep.py [--max 256] [--precision f16x2|fp32]
"""
import argparse
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import tf_raft_b200 as T
from tf_raft_b200 import _lib


def ev_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--max', type=int, default=256)
    ap.add_argument('--precision', default='f16x2', choices=['f16x2', 'fp32'])
    args = ap.parse_args()
    print(f'{"g":>4} {"N":>6} {"pyramid MB":>11} {"K1 ms":>8} {"K1 GB/s":>8} {"K2 us":>8} {"K2 GB/s":>8} {"K2(int) us":>10}')
    for g in (32, 48, 64, 96, 128, 192, 256):
        if g > args.max:
            break
        n = g * g
        pyr_bytes = 4 * sum(n * (g >> l) * (g >> l) for l in range(4))
        if pyr_bytes > 0.8 * torch.cuda.get_device_properties(0).total_memory:
            print(f'{g:4d}: pyramid {pyr_bytes/1e9:.0f} GB does not fit')
            continue
        gen = torch.Generator().manual_seed(g)
        f1 = torch.randn((1, g, g, 256), generator=gen).cuda()
        f2 = torch.randn((1, g, g, 256), generator=gen).cuda()
        cb = T.CorrBlock(f1, f2, 4, 4, precision=args.precision)
        ptrs = _lib.ptr_array(cb.corr_pyramid)

        def build():
            _lib.check(_lib.lib().raft_b200_corr_pyramid_build(_lib.ptr(f1), _lib.ptr(f2), 1, g, g, 256, 4, ptrs, _lib.ptr(cb._ws),
                                                               cb._ws.numel(), cb.precision, _lib.stream()), 'corr_pyramid_build')
        grid = T.coords_grid(1, g, g, f1.device)
        jit = torch.from_numpy(np.random.default_rng(2).uniform(-8, 8, (1, g, g, 2)).astype(np.float32)).cuda()
        out = torch.empty((1, g, g, 324), device=f1.device)

        def lookup(coords):
            def run():
                _lib.check(_lib.lib().raft_b200_corr_lookup(ptrs, _lib.ptr(coords), 1, g, g, 4, 4, _lib.ptr(out), 324, _lib.stream()),
                           'corr_lookup')
            return run
        reps = 20 if g <= 96 else 5
        t1 = ev_time(build, reps)
        t2 = ev_time(lookup((grid + jit).contiguous()), reps * 4)
        t2i = ev_time(lookup(grid), reps * 4)
        k1_bytes = pyr_bytes + 2 * n * 256 * 4
        k2_bytes = n * 2904
        print(f'{g:4d} {n:6d} {pyr_bytes/1e6:11.1f} {t1*1e3:8.3f} {k1_bytes/t1/1e9:8.0f} {t2*1e6:8.1f} {k2_bytes/t2/1e9:8.0f} {t2i*1e6:10.1f}')
        del cb, f1, f2, out
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
