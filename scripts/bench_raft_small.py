"""Cost of the original PyTorch RAFT-small (SmallRAFT(conventions='pytorch', blocks='bottleneck')) against tf-raft's
SmallRAFT, on one GPU:

  * model: pairs/s of inference (f16x2, CUDA graph, last_only) at 448x512 x 12 iterations (batch 4) and 440x1024 x 32
    iterations (batch 1), the two models alternating, medians of rounds;
  * encode: milliseconds of the inference encode alone (raft_b200_encode_pair: fnet on both images, cnet on the
    first), CUDA events, the two models alternating, and the kernels it launches;
  * upflow8: kernel microseconds of the align-corners upflow8 against the half-pixel one at 56x64 (batch 4) and 55x128
    (batch 1): CUDA events around the replay of a CUDA graph of 100 calls, so that no host time enters, alternating.
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

MODELS = {'tf-raft-small': {}, 'raft-small-pytorch': {'conventions': 'pytorch', 'blocks': 'bottleneck'}}


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return torch.cuda.get_device_name()


def _images(b, H, W):
    rng = np.random.default_rng(0)
    im1 = torch.from_numpy(rng.uniform(0, 255, (b, H, W, 3)).astype(np.float32)).cuda()
    return im1, torch.roll(im1, 4, dims=2).contiguous()


def _models(T, iters, use_graph):
    return {name: T.SmallRAFT(precision='f16x2', iters_pred=iters, use_graph=use_graph, device='cuda', seed=1, **kw)
            for name, kw in MODELS.items()}


def pairs_per_s(T, b, H, W, iters, steps, rounds):
    im1, im2 = _images(b, H, W)
    models = _models(T, iters, True)
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


def _events(fn, reps):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def encode_ms(T, b, H, W, reps, rounds):
    from tf_raft_b200 import _lib
    im1, im2 = _images(b, H, W)
    models = _models(T, 1, False)
    res = {c: [] for c in models}
    launches = {}
    for c, m in models.items():
        m._encode_pair(im1, im2)
        _lib.launch_count_reset()
        m._encode_pair(im1, im2)
        launches[c] = _lib.launch_count()
    for _ in range(rounds):
        for c, m in models.items():
            res[c].append(_events(lambda: m._encode_pair(im1, im2), reps))
    return {c: {'ms': float(np.median(v)), 'launches': launches[c]} for c, v in res.items()}


def upflow8_us(b, h, w, reps, rounds):
    from tf_raft_b200 import _lib
    flow = torch.randn(b, h, w, 2, device='cuda', generator=torch.Generator(device='cuda').manual_seed(0)) * 5
    out = torch.empty(b, 8 * h, 8 * w, 2, device='cuda')
    graphs = {}
    for k, fn in (('half_pixel', 'upflow8'), ('align_corners', 'upflow8_align_corners')):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            _lib.call(fn, flow.device, _lib.ptr(flow), b, h, w, _lib.ptr(out))
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(reps):
                _lib.call(fn, flow.device, _lib.ptr(flow), b, h, w, _lib.ptr(out))
        graphs[k] = g
    res = {k: [] for k in graphs}
    for _ in range(rounds):
        for k, g in graphs.items():
            res[k].append(1e3 * _events(g.replay, 1) / reps)
    return {k: float(np.median(v)) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_raft_small.py measures on a CUDA device; none is available')
    import tf_raft_b200 as T
    result = {'card': card(),
              'pairs_per_s': {'448x512_b4_12it': pairs_per_s(T, 4, 448, 512, 12, a.steps, a.rounds),
                              '440x1024_b1_32it': pairs_per_s(T, 1, 440, 1024, 32, a.steps, a.rounds)},
              'encode_ms': {'448x512_b4': encode_ms(T, 4, 448, 512, 20, a.rounds),
                            '440x1024_b1': encode_ms(T, 1, 440, 1024, 20, a.rounds)},
              'upflow8_us': {'4x56x64': upflow8_us(4, 56, 64, 100, a.rounds),
                             '1x55x128': upflow8_us(1, 55, 128, 100, a.rounds)}}
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'bench_raft_small.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
