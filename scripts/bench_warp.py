"""Flow warping and composition throughput, and what chaining costs in `RAFT.track_video`.

    python scripts/bench_warp.py --out DIR [--calls 50 --windows 5 --clips 2 --frames 8 --iters 12]

Kernels, on seeded inputs already on the GPU, CUDA events around device-synchronised windows of `--calls` calls to
the library (preallocated outputs, so only the kernel and its launch are timed), median and best of `--windows`:
  * raft_b200_warp, float32 bilinear at C = 1, 3 and 64, float32 nearest at C = 3, and uint8 nearest at C = 1;
  * raft_b200_compose_flow with both masks;
each at batch 8 x 436 x 1024 (Sintel's frame size) and batch 1 x 1080 x 1920.  Beside each time, the bytes the kernel
must move at least (flow, output and mask once, the source once) over that time.
Tracking: RAFT with the tests' seeded weights, f16x2, eager, on B synthetic clips of T frames at 440 x 1024 (Sintel's
436 rows padded to a multiple of 8): seconds per clip batch of predict_video(bidirectional=True) and of
track_video in each direction, the two alternating over `--rounds` rounds, medians.
The GPU's name, power limit and maximum SM clock are read (nvidia-smi, query only) in the same run: one JSON line on
stdout and in DIR/bench_warp.json.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import torch  # noqa: E402

import cases  # noqa: E402
from oracle import weights  # noqa: E402
import tf_raft_b200 as T  # noqa: E402
from tf_raft_b200 import _lib  # noqa: E402


def gpu_info():
    try:
        res = subprocess.run(['nvidia-smi', f'--id={torch.cuda.current_device()}',
                              '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=60)
        return res.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f'nvidia-smi unavailable: {e}'


def timed(fn, args):
    for _ in range(3):
        fn()
    windows = []
    for _ in range(args.windows):
        torch.cuda.synchronize()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(args.calls):
            fn()
        end.record()
        torch.cuda.synchronize()
        windows.append(start.elapsed_time(end) / args.calls)
    return statistics.median(windows), min(windows)


def flow_field(b, h, w, g):
    """A smooth flow of up to ~20 px with a tenth of the landings outside the frame."""
    yy, xx = torch.meshgrid(torch.arange(h, device='cuda'), torch.arange(w, device='cuda'), indexing='ij')
    fx = 20 * torch.sin(yy / 37.0 + torch.rand(b, 1, 1, device='cuda', generator=g)) * torch.cos(xx / 53.0)
    fy = 15 * torch.cos(xx / 41.0 + torch.rand(b, 1, 1, device='cuda', generator=g))
    return torch.stack([fx, fy], -1).float().contiguous()


def bench_kernels(args):
    g = torch.Generator(device='cuda').manual_seed(0)
    out = {}
    for b, h, w in ((8, 436, 1024), (1, 1080, 1920)):
        flow = flow_field(b, h, w, g)
        occ = torch.empty((b, h, w), dtype=torch.uint8, device='cuda')
        npix = b * h * w
        entry = {}
        for name, c, dtype, mode in (('f32_bilinear_c1', 1, 'f32', 'bilinear'), ('f32_bilinear_c3', 3, 'f32', 'bilinear'),
                                     ('f32_bilinear_c64', 64, 'f32', 'bilinear'), ('f32_nearest_c3', 3, 'f32', 'nearest'),
                                     ('u8_nearest_c1', 1, 'u8', 'nearest')):
            if dtype == 'f32':
                src = torch.rand((b, h, w, c), device='cuda', generator=g)
            else:
                src = torch.randint(0, 255, (b, h, w, c), dtype=torch.uint8, device='cuda', generator=g)
            dst = torch.empty_like(src)
            esz = src.element_size()
            code = _lib.WARP_F32 if dtype == 'f32' else _lib.WARP_U8

            def run():
                _lib.call('warp', src.device, _lib.ptr(src), code, h, w, c, _lib.ptr(flow), b, h, w,
                          _lib.WARP_MODES[mode], 0.0, _lib.ptr(dst), _lib.ptr(occ))
            med, best = timed(run, args)
            nbytes = npix * (8 + 1 + 2 * c * esz)
            entry[name] = {'ms_median': round(med, 4), 'ms_best': round(best, 4),
                           'min_bytes_GBps_at_median': round(nbytes / (med * 1e-3) / 1e9, 1)}
            del src, dst
        f2 = flow_field(b, h, w, g)
        o1 = (torch.rand((b, h, w), device='cuda', generator=g) < 0.1).to(torch.uint8)
        o2 = (torch.rand((b, h, w), device='cuda', generator=g) < 0.1).to(torch.uint8)
        acc = torch.empty_like(flow)

        def run_compose():
            _lib.call('compose_flow', flow.device, _lib.ptr(flow), _lib.ptr(f2), _lib.ptr(o1), _lib.ptr(o2), b, h, w,
                      _lib.ptr(acc), _lib.ptr(occ))
        med, best = timed(run_compose, args)
        nbytes = npix * (8 + 8 + 1 + 1 + 8 + 1)
        entry['compose_flow'] = {'ms_median': round(med, 4), 'ms_best': round(best, 4),
                                 'min_bytes_GBps_at_median': round(nbytes / (med * 1e-3) / 1e9, 1)}
        out[f'{b}x{h}x{w}'] = entry
    return out


def bench_tracking(args):
    B, n, H, W = args.clips, args.frames, 440, 1024
    model = T.RAFT(iters=args.iters, iters_pred=args.iters, precision='f16x2')
    model.load_params(weights.init_params('raft', 1234, bias_scale=0.05, norm_jitter=0.1))
    frames = [torch.from_numpy(cases.images(B, H, W, 700 + t, 700 + t)[0]).cuda() for t in range(n)]

    def video():
        for _ in model.predict_video(frames, bidirectional=True):
            pass

    def track(direction):
        def run():
            for _ in model.track_video(frames, direction=direction):
                pass
        return run

    runs = {'predict_video_bidirectional': video, 'track_video_forward': track('forward'),
            'track_video_backward': track('backward')}
    for fn in runs.values():
        fn()
    times = {k: [] for k in runs}
    for _ in range(args.rounds):
        for k, fn in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    res = {k: round(statistics.median(v), 4) for k, v in times.items()}
    base = res['predict_video_bidirectional']
    return {'clips': B, 'frames': n, 'height': H, 'width': W, 'iters_pred': args.iters, 's_per_clip_batch': res,
            'overhead_pct': {k: round(100 * (v / base - 1), 2) for k, v in res.items() if k != 'predict_video_bidirectional'},
            'times_s': {k: [round(x, 4) for x in v] for k, v in times.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--calls', type=int, default=50)
    ap.add_argument('--windows', type=int, default=5)
    ap.add_argument('--clips', type=int, default=2)
    ap.add_argument('--frames', type=int, default=8)
    ap.add_argument('--iters', type=int, default=12)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_warp.py needs a CUDA device')
    os.makedirs(args.out, exist_ok=True)
    result = {'metric': 'ms per kernel call; s per tracked clip batch', 'gpu': gpu_info(),
              'device': torch.cuda.get_device_name(), 'kernels': bench_kernels(args), 'tracking': bench_tracking(args)}
    line = json.dumps(result)
    print(line)
    with open(os.path.join(args.out, 'bench_warp.json'), 'w') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
