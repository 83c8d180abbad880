"""Video inference throughput at the Sintel geometry: per-pair calls against predict_video (cold and warm start), one
direction and both directions with occlusion masks.

    python scripts/bench_video.py --out DIR [--clips 4 --frames 13 --height 448 --width 1024 --iters 24 12 --repeats 3]

B seeded synthetic clips of T frames, RAFT with the seeded weights of the tests, the f16x2 path, eager launches.  For every
`iters_pred` it times, over the whole sequence (B * (T - 1) flows):
  * per_pair:   model([f_{t-1}, f_t], training=False, last_only=True) for t = 1 .. T-1 (three image encodes per pair);
  * video_cold: model.predict_video(frames, warm_start=False) (two image encodes per pair);
  * video_warm: model.predict_video(frames, warm_start=True) (two encodes plus the forward interpolation);
and both directions of every pair with their forward-backward occlusion masks:
  * per_pair_both:    model([f_{t-1}, f_t]) and model([f_t, f_{t-1}]) plus fb_occlusion (six image encodes per pair);
  * video_bidir_cold: model.predict_video(frames, warm_start=False, bidirectional=True) (two encodes per pair, one
                      batch-2B loop);
  * video_bidir_warm: the same with warm_start=True (one forward interpolation of both halves per pair).
Rates are flows per second (B * (T - 1) / window) for the one-direction modes and bidirectional pairs per second
(B * (T - 1) / window, each pair two flows and two masks) for the others, from CUDA events around device-synchronised
windows, after one untimed pass of every mode; median and best of `--repeats` windows.  Also timed: one fnet and one cnet
call on B frames, the forward_interpolate kernel on (B, H/8, W/8) and (1, 216, 216) flows, and fb_occlusion on
(B, H, W) flows.  The GPU's name, power limit and maximum SM clock are read (nvidia-smi, query only) in the same run and
written beside the numbers: one JSON line on stdout and in DIR/bench_video.json.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import numpy as np  # noqa: E402
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


def timed(fn, repeats):
    """Milliseconds of fn() per window: CUDA events around a device-synchronised window, one window per repeat."""
    out = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        fn()
        end.record()
        end.synchronize()
        out.append(start.elapsed_time(end))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True, help='directory for bench_video.json')
    ap.add_argument('--clips', type=int, default=4)
    ap.add_argument('--frames', type=int, default=13)
    ap.add_argument('--height', type=int, default=448)
    ap.add_argument('--width', type=int, default=1024)
    ap.add_argument('--iters', type=int, nargs='+', default=[24, 12])
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_video.py needs a GPU'
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 (H100) device'
    B, n, H, W = args.clips, args.frames, args.height, args.width
    flows = B * (n - 1)
    frames = [torch.from_numpy(cases.images(B, H, W, 500 + t, 500 + t)[0]).cuda() for t in range(n)]
    model = T.RAFT(precision='f16x2')
    model.load_params(weights.init_params('raft', 1234))

    def per_pair():
        for t in range(1, n):
            model([frames[t - 1], frames[t]], training=False, last_only=True)

    def per_pair_both():
        for t in range(1, n):
            fw = model([frames[t - 1], frames[t]], training=False, last_only=True)[-1]
            bw = model([frames[t], frames[t - 1]], training=False, last_only=True)[-1]
            T.fb_occlusion(fw, bw)

    def video(warm, bidirectional=False):
        def run():
            for _ in model.predict_video(frames, warm_start=warm, bidirectional=bidirectional):
                pass
        return run

    result = dict(metric='flows/s (B clips x (T-1) pairs per window)', gpu=gpu_info(), device=torch.cuda.get_device_name(),
                  clips=B, frames=n, height=H, width=W, precision='f16x2', repeats=args.repeats, modes={})
    for iters in args.iters:
        model.iters_pred = iters
        modes = {'per_pair': per_pair, 'video_cold': video(False), 'video_warm': video(True),
                 'per_pair_both': per_pair_both, 'video_bidir_cold': video(False, True),
                 'video_bidir_warm': video(True, True)}
        for fn in modes.values():                                  # warm-up: every shape and mode once
            fn()
        # the same sequence's last flow from the two cold paths, as a cross-check (bit-identical on the native encoders)
        last_pair = model([frames[-2], frames[-1]], training=False, last_only=True)[-1].clone()
        last_video = list(model.predict_video(frames[-2:], warm_start=False))[-1]
        row = {'cold_video_equals_per_pair': bool(torch.equal(last_pair, last_video))}
        # and both directions: the cold bidirectional video against predict_bidirectional and the two per-pair flows
        both = [x.clone() for x in model.predict_bidirectional([frames[-2], frames[-1]])]
        last_bidir = list(model.predict_video(frames[-2:], warm_start=False, bidirectional=True))[-1]
        last_bw = model([frames[-1], frames[-2]], training=False, last_only=True)[-1]
        row['cold_bidir_video_equals_per_pair'] = bool(
            all(torch.equal(a, b) for a, b in zip(both, last_bidir)) and torch.equal(both[0], last_pair)
            and torch.equal(both[1], last_bw))
        for name, fn in modes.items():
            ms = timed(fn, args.repeats)
            unit = 'bidir_pairs' if name in ('per_pair_both', 'video_bidir_cold', 'video_bidir_warm') else 'flows'
            row[name] = {f'{unit}_per_s_median': round(flows / (statistics.median(ms) / 1e3), 2),
                         f'{unit}_per_s_best': round(flows / (min(ms) / 1e3), 2),
                         'window_ms': [round(m, 2) for m in ms]}
        result['modes'][f'iters_pred={iters}'] = row

    enc = {}
    for name, net in (('fnet', model.fnet), ('cnet', model.cnet)):
        net(frames[0], training=False, raw_image=True)
        ms = timed(lambda: [net(frames[0], training=False, raw_image=True) for _ in range(10)], args.repeats)
        enc[f'{name}_ms_per_call_on_{B}_frames'] = round(statistics.median(ms) / 10, 3)
    result['encoders'] = enc

    fi = {}
    rng = np.random.default_rng(3)
    for b, h, w in ((B, H // 8, W // 8), (1, 216, 216)):
        flow = torch.from_numpy(rng.uniform(-3, 3, (b, h, w, 2)).astype(np.float32)).cuda()
        for _ in range(3):
            T.forward_interpolate(flow)
        reps = 20 if h * w < 20000 else 5
        ms = timed(lambda: [T.forward_interpolate(flow) for _ in range(reps)], args.repeats)
        fi[f'{b}x{h}x{w}_ms'] = round(statistics.median(ms) / reps, 4)
    result['forward_interpolate'] = fi

    fw, bw = (torch.from_numpy(rng.uniform(-3, 3, (B, H, W, 2)).astype(np.float32)).cuda() for _ in range(2))
    for _ in range(3):
        T.fb_occlusion(fw, bw)
    ms = timed(lambda: [T.fb_occlusion(fw, bw) for _ in range(50)], args.repeats)
    # the kernel alone: raw entry-point launches into preallocated masks, queued faster than they run
    occ = [torch.empty((B, H, W), dtype=torch.bool, device='cuda') for _ in range(2)]
    args_c = [_lib.ptr(fw), _lib.ptr(bw), B, H, W, 0.01, 0.5, _lib.ptr(occ[0]), _lib.ptr(occ[1]), _lib.stream()]
    ms_k = timed(lambda: [_lib.lib().raft_b200_fb_occlusion(*args_c) for _ in range(200)], args.repeats)
    result['fb_occlusion'] = {f'{B}x{H}x{W}_ms_per_call': round(statistics.median(ms) / 50, 4),
                              f'{B}x{H}x{W}_ms_kernel': round(statistics.median(ms_k) / 200, 4)}

    line = json.dumps(result)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'bench_video.json'), 'w') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
