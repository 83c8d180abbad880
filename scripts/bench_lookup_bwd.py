"""Time raft_b200_corr_lookup_backward of one or more builds of the library, alternating them in one process.

    python scripts/bench_lookup_bwd.py --lib A.so [--lib B.so ...] [--rounds 5] [--calls 200] [--out DIR]

The entry point is called through ctypes from each library path given, so an older build (another commit's .so) is timed
by the same script on the same buffers.  Shapes (RAFT's 4-level pyramid over a 368 x 496 Chairs crop, 46 x 62 queries):
  chairs : B = 4, r = 4 (the supervised step);
  unsup  : B = 8, r = 4 (the self-supervised step runs both directions, 2B);
  small  : B = 4, r = 3 (SmallRAFT).
Coordinates are the query grid plus a smooth flow of a few pixels with sub-pixel detail (the middle of training); the
pyramid and grad_out are seeded normals.  Each round times `--calls` back-to-back launches per library with CUDA events
(the accumulators are not re-zeroed: the kernel's work does not depend on their values); the median per-call time over
the rounds is reported with the card's name and power limit.  One JSON line on stdout, and DIR/bench_lookup_bwd.json
with --out."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess

import numpy as np
import torch

SHAPES = {'chairs': (4, 46, 62, 4), 'unsup': (8, 46, 62, 4), 'small': (4, 46, 62, 3)}
LEVELS = 4


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else 'unknown'


def load(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    vp, i = ctypes.c_void_p, ctypes.c_int
    fn = lib.raft_b200_corr_lookup_backward
    fn.restype = i
    fn.argtypes = [ctypes.POINTER(vp), vp, vp, i, i, i, i, i, vp, ctypes.POINTER(vp), vp]
    return fn


def case(b, h, w, r, seed=0):
    rng = np.random.default_rng(seed)
    gy, gx = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing='ij')
    fx = 6 * np.sin(gy / 9 + 0.3) + 3 * np.cos(gx / 13) + rng.normal(0, 0.4, (b, h, w))
    fy = 4 * np.cos(gx / 11 - 0.2) - 2 * np.sin(gy / 7) + rng.normal(0, 0.4, (b, h, w))
    coords = torch.from_numpy(np.stack([gx + fx, gy + fy], axis=-1).astype(np.float32)).cuda()
    gen = torch.Generator(device='cuda').manual_seed(seed)
    nq = b * h * w
    pyr = [torch.randn((nq, h >> l, w >> l, 1), generator=gen, device='cuda') for l in range(LEVELS)]
    g = torch.randn((b, h, w, LEVELS * (2 * r + 1) ** 2), generator=gen, device='cuda') * 1e-3
    gpyr = [torch.zeros_like(p) for p in pyr]
    gc = torch.zeros_like(coords)
    arr = lambda ts: (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
    return (arr(pyr), ctypes.c_void_p(coords.data_ptr()), ctypes.c_void_p(g.data_ptr()), b, h, w, LEVELS, r,
            ctypes.c_void_p(gc.data_ptr()), arr(gpyr)), (pyr, g, gpyr, gc, coords)


def time_calls(fn, args, calls, stream):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        assert fn(*args, stream) == 0
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', action='append', required=True, help='libraft_b200.so to time (repeatable)')
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--calls', type=int, default=200)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_lookup_bwd needs a CUDA device')
    fns = {p: load(p) for p in args.lib}
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    res = {'card': card(), 'calls_per_round': args.calls, 'shapes': {}}
    for name, (b, h, w, r) in SHAPES.items():
        cargs, keep = case(b, h, w, r)
        for fn in fns.values():                                      # warm-up
            time_calls(fn, cargs, 5, stream)
        ms = {p: [] for p in fns}
        for _ in range(args.rounds):
            for p, fn in fns.items():
                ms[p].append(time_calls(fn, cargs, args.calls, stream))
        res['shapes'][name] = {'B': b, 'h': h, 'w': w, 'radius': r, 'levels': LEVELS,
                               'ms_per_call': {p: {'median': round(statistics.median(v), 4), 'min': round(min(v), 4),
                                                   'max': round(max(v), 4)} for p, v in ms.items()}}
        del keep
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_lookup_bwd.json'), 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
