"""Training-step throughput with train_precision 'fp32' and 'f16x2' at the Chairs config (RAFT, batch 4, 368 x 496,
12 iterations): bare `train_step` pairs/s, the two modes alternating in one run, several windows each (medians and
spreads); the card's name and power limit; in a separate torch.profiler run of the f16x2 step, the step's GPU time by
kind; and the weight-gradient call's achieved rate at two layer shapes.

    python scripts/bench_train_tc.py [--windows 3] [--steps 10] [--warmup 3] [--out DIR]

Writes DIR/bench_train_tc.json (default: a temporary directory) and prints one JSON line."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))

B, H, W, ITERS = 4, 368, 496, 12


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else 'unknown'


def model(train_precision):
    from tf_raft_b200 import RAFT
    from tf_raft_b200.train import AdamW
    m = RAFT(iters=ITERS, seed=0)
    m.compile(optimizer=AdamW(weight_decay=1e-4, learning_rate=1e-4), clip_norm=1.0, train_precision=train_precision)
    return m


def batch(seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    im1 = torch.rand((B, H, W, 3), generator=g, device='cuda') * 255
    im2 = torch.roll(im1, shifts=(3, 5), dims=(1, 2))
    flow = torch.randn((B, H, W, 2), generator=g, device='cuda') * 4
    return im1, im2, flow, torch.ones((B, H, W), device='cuda')


def window(m, data, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        m.train_step(data)
    torch.cuda.synchronize()
    return steps * B / (time.perf_counter() - t0)


def kind(name):
    if 'conv_wgrad_tc_kernel' in name or 'wgrad_reduce' in name:
        return 'tensor-core weight gradient'
    if 'conv_tc_kernel' in name:
        return 'tensor-core forward + input gradient (conv_tc_kernel)'
    if any(k in name for k in ('train_split', 'absmax', 'pack_weights', 'wgrad_scale', 'weight_scale')):
        return 'tensor-core operand preparation (split, pack, scale)'
    if any(k in name for k in ('im2col', 'col2im', 'gemm', 'Gemm', 'conv', 'sm90_xmma', 'cutlass')):
        return 'library convolutions and GEMMs'
    return 'everything else'


def profile(m, data):
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        m.train_step(data)
        torch.cuda.synchronize()
    by = {}
    for e in p.key_averages():
        t = getattr(e, 'device_time_total', None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            by[kind(e.key)] = by.get(kind(e.key), 0.0) + t / 1e3
    return {k: round(v, 3) for k, v in sorted(by.items(), key=lambda kv: -kv[1])}


def wgrad_rate(shape, reps=20):
    """Achieved rate of raft_b200_conv_tc_backward without the input gradient (split, pack, wgrad kernel, reduction):
    useful FLOPs 2 * B*H*W * kh*kw * cin * cout over CUDA-event time."""
    from tf_raft_b200 import _lib
    b, h, w, cin, kh, kw, cout = shape
    x = torch.randn((b, h, w, cin), device='cuda')
    k = torch.randn((kh, kw, cin, cout), device='cuda') * 0.1
    bias = torch.zeros(cout, device='cuda')
    g = torch.randn((b, h, w, cout), device='cuda') * 1e-6
    need = ctypes.c_size_t()
    _lib.call('conv_tc_forward', x.device, None, None, None, *shape, None, None, None, ctypes.byref(need))
    ws = _lib.workspace(need.value, x.device)
    nb = ctypes.byref(ctypes.c_size_t(ws.numel()))
    planes = torch.empty(2 * b * h * w * ((cin + 63) // 64 * 64) + 128, dtype=torch.float16, device='cuda')
    out = torch.empty((b, h, w, cout), device='cuda')
    dk = torch.empty_like(k)
    _lib.call('conv_tc_forward', x.device, _lib.ptr(x), _lib.ptr(k), _lib.ptr(bias), *shape, _lib.ptr(out),
              _lib.ptr(planes), _lib.ptr(ws), nb)
    call = lambda: _lib.call('conv_tc_backward', x.device, _lib.ptr(planes), _lib.ptr(k), _lib.ptr(g), *shape, None,
                             _lib.ptr(dk), _lib.ptr(ws), nb)
    for _ in range(3):
        call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    flops = 2.0 * b * h * w * kh * kw * cin * cout
    return {'shape': list(shape), 'ms': round(ms, 4), 'useful_tflops': round(flops / ms / 1e9, 2),
            'three_pass_bound_tflops': round(989.0 / 3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--windows', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_train_tc needs a CUDA device')
    from tf_raft_b200 import build
    build.build()
    gpu = card()
    data = batch()
    models = {mode: model(mode) for mode in ('fp32', 'f16x2')}
    for m in models.values():
        for _ in range(args.warmup):
            m.train_step(data)
    rates = {mode: [] for mode in models}
    for _ in range(args.windows):
        for mode, m in models.items():
            rates[mode].append(window(m, data, args.steps))
    summary = {mode: {'median_pairs_per_s': round(statistics.median(r), 3), 'min': round(min(r), 3),
                      'max': round(max(r), 3), 'windows': [round(v, 3) for v in r]} for mode, r in rates.items()}
    breakdown = profile(models["f16x2"], data)
    wgrad = [wgrad_rate(s) for s in ((8, 184, 248, 64, 3, 3, 64), (4, 46, 62, 384, 1, 5, 128))]
    res = {'card': gpu, 'config': f'RAFT batch {B} {H}x{W} iters {ITERS}', 'train_step': summary,
           'speedup_f16x2_over_fp32': round(summary['f16x2']['median_pairs_per_s'] / summary['fp32']['median_pairs_per_s'], 3),
           'f16x2_step_gpu_ms_by_kind': breakdown, 'wgrad_call': wgrad}
    out_dir = args.out or tempfile.mkdtemp(prefix='bench_train_tc_')
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, 'bench_train_tc.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
