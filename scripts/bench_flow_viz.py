"""Flow colour-wheel visualisation: raft_b200_flow_to_image's device time and `flow_to_image` end to end.

    python scripts/bench_flow_viz.py --out DIR [--launches 200 --calls 50]

Seeded smooth float32 flows already on the GPU, at 436x1024 and 448x1024, batches of 1 and 16:
  * kernel_ms: CUDA events around `--launches` back-to-back calls of the C entry point (zeroing of the status and
    reduction words, flow_radmax_kernel, flow_colour_kernel) on preallocated buffers after a warm-up, per batch;
  * e2e_ms_per_frame: `flow_to_image(flow).cpu()` per frame, wall clock over `--calls` calls: the Python checks, the
    launches, the read of the status words and the D2H copy of the uint8 image;
  * numpy_ms_per_frame: the NumPy restatement (oracle/flow_viz_np.py) on the host, the same frame, for scale.
The GPU's name, power limit and maximum SM clock are read (nvidia-smi, query only) in the same run: one JSON line on
stdout and in DIR/bench_flow_viz.json.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import flow_viz_np as F  # noqa: E402
from tf_raft_b200 import _lib  # noqa: E402
from tf_raft_b200.datasets import flow_to_image  # noqa: E402


def gpu_info():
    try:
        res = subprocess.run(['nvidia-smi', f'--id={torch.cuda.current_device()}',
                              '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=60)
        return res.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f'nvidia-smi unavailable: {e}'


def kernel_ms(flow, launches):
    b, h, w, _ = flow.shape
    image = torch.empty((b, h, w, 3), dtype=torch.uint8, device='cuda')
    work = torch.empty(b, dtype=torch.int32, device='cuda')
    status = torch.empty(b, dtype=torch.int32, device='cuda')
    u = flow.reshape(-1)

    def call():
        _lib.check(_lib.lib().raft_b200_flow_to_image(_lib.ptr(u), _lib.ptr(u[1:]), 2, b, h, w, 0, 0.0, 1, None, 0,
                                                      _lib.ptr(image), _lib.ptr(work), _lib.ptr(status), _lib.stream()))
    for _ in range(20):
        call()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        call()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--calls', type=int, default=50)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    rng = np.random.default_rng(0)
    result = {'gpu': gpu_info(), 'device': torch.cuda.get_device_name(), 'numpy': np.__version__, 'cases': {}}
    for h, w in ((436, 1024), (448, 1024)):
        frames = np.stack([F._smooth(rng, h, w, 20.0) for _ in range(16)])
        for b in (1, 16):
            flow = torch.from_numpy(frames[:b]).cuda()
            k = kernel_ms(flow, args.launches)
            for _ in range(5):
                flow_to_image(flow).cpu()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.calls):
                flow_to_image(flow).cpu()
            e2e = (time.perf_counter() - t0) * 1e3 / args.calls / b
            result['cases'][f'{h}x{w}_B{b}'] = {'kernel_ms': round(k, 4), 'kernel_ms_per_frame': round(k / b, 4),
                                                'e2e_ms_per_frame': round(e2e, 4)}
        t0 = time.perf_counter()
        for _ in range(3):
            F.flow_to_image(frames[0])
        result['cases'][f'{h}x{w}_numpy_ms_per_frame'] = round((time.perf_counter() - t0) * 1e3 / 3, 1)
    line = json.dumps(result)
    print(line)
    with open(os.path.join(args.out, 'bench_flow_viz.json'), 'w') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
