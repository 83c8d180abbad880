"""The encode phase of the inference forward: fnet on both images, cnet and the context split, the correlation pyramid --
serially (the separate fnet / cnet / CorrBlock calls) and as the concurrent branches of raft_b200_encode_pair.

    python scripts/bench_encode.py --out DIR [--batch 4 --height 448 --width 512 --reps 20 --repeats 5]

RAFT with bench.py's seeded weights, the f16x2 path.  Each timed item is captured once into a CUDA graph (as bench.py
replays the whole forward) and replayed `--reps` times per window; CUDA events around device-synchronised windows,
median and best of `--repeats` windows, in ms per call:
  * fnet:        fnet([image1, image2]), batch 2B;
  * cnet:        cnet(image1) and the context split, batch B;
  * pyramid:     raft_b200_corr_pyramid_build on fixed buffers;
  * serial:      the whole phase as the separate fnet / cnet calls + CorrBlock (what the forward ran before
                 raft_b200_encode_pair);
  * concurrent:  the whole phase as RAFT._encode_pair + CorrBlock;
  * serial_eager / concurrent_eager: the same two without a graph (host launch cost included).
A separate torch.profiler run of eager serial and concurrent phases gives the device time of every kernel, summed by kind:
conv (conv_tc_kernel), norm (statistics, finalisation, apply), stem (image normalisation, stem im2col), pyramid
(corr_prep / corr_tc), split, memset.  conv is tensor-bound, norm / stem / split / memset are HBM passes.  The profiler's
key-average table goes to DIR/bench_encode_profile.txt.  The GPU's name, power limit and maximum SM clock are read
(nvidia-smi, query only) in the same run: one JSON line on stdout and in DIR/bench_encode.json.
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


def windows(fn, reps, repeats):
    """ms per fn() call: CUDA events around device-synchronised windows of `reps` calls; (median, best)."""
    out = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / reps)
    return statistics.median(out), min(out)


def graphed(fn):
    """fn captured into a CUDA graph after two eager warm-up calls on a side stream; returns the replay."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph.replay


KINDS = (('conv', ('conv_tc_kernel',)), ('norm', ('norm_stats', 'norm_final', 'norm_apply')),
         ('stem', ('image_norm', 'stem_im2col')), ('pyramid', ('corr_prep', 'corr_tc')), ('split', ('context_split',)),
         ('memset', ('memset', 'Memset')))


def kind(name):
    for k, keys in KINDS:
        if any(s in name for s in keys):
            return k
    return 'other'


def profile(fn, calls, path):
    """Device time per call of every kernel kind (ms) from a torch.profiler run of `calls` eager calls."""
    from torch.profiler import ProfilerActivity, profile as prof
    fn()
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    sums = {}
    for ev in p.key_averages():
        t = getattr(ev, 'device_time_total', None)
        if t is None:
            t = ev.cuda_time_total
        if t:
            sums[kind(ev.key)] = sums.get(kind(ev.key), 0.0) + t / 1e3 / calls
    with open(path, 'w') as f:
        f.write(p.key_averages().table(sort_by='device_time_total', row_limit=40))
    return {k: round(v, 4) for k, v in sorted(sums.items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--height', type=int, default=448)
    ap.add_argument('--width', type=int, default=512)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=5)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    assert torch.cuda.is_available() and _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, \
        'needs an sm_90 GPU'
    B, H, W = args.batch, args.height, args.width
    model = T.RAFT(iters=12, iters_pred=12, precision='f16x2')
    model.load_params(weights.init_params('raft', 1234))
    a, b = (torch.from_numpy(x).cuda() for x in cases.images(B, H, W, 0, 1))

    fmap1, fmap2, _, _ = model._encode(a, b, False)
    cb = T.CorrBlock(fmap1, fmap2, 4, 4, precision='f16x2')
    pyr = _lib.ptr_array(cb.corr_pyramid)

    def pyramid():
        _lib.check(_lib.lib().raft_b200_corr_pyramid_build(
            _lib.ptr(fmap1), _lib.ptr(fmap2), B, H // 8, W // 8, 256, 4, pyr, _lib.ptr(cb._ws), cb._ws.numel(),
            cb.precision, _lib.stream()), 'corr_pyramid_build')

    def serial():
        f1, f2 = model.fnet([a, b], training=False, raw_image=True)
        model._context(a, False)
        T.CorrBlock(f1, f2, 4, 4, precision='f16x2')

    def concurrent():
        f1, f2, _, _ = model._encode_pair(a, b)
        T.CorrBlock(f1, f2, 4, 4, precision='f16x2')

    items = {'fnet': lambda: model.fnet([a, b], training=False, raw_image=True),
             'cnet': lambda: model._context(a, False), 'pyramid': pyramid, 'serial': serial, 'concurrent': concurrent}
    ms = {}
    for name, fn in items.items():
        med, best = windows(graphed(fn), args.reps, args.repeats)
        ms[name] = {'median': round(med, 4), 'best': round(best, 4)}
    for name, fn in (('serial_eager', serial), ('concurrent_eager', concurrent)):
        fn()
        med, best = windows(fn, args.reps, args.repeats)
        ms[name] = {'median': round(med, 4), 'best': round(best, 4)}
    kinds = {'serial': profile(serial, 5, os.path.join(args.out, 'bench_encode_profile.txt')),
             'concurrent': profile(concurrent, 5, os.path.join(args.out, 'bench_encode_profile_concurrent.txt'))}
    hbm = sum(v for k, v in kinds['serial'].items() if k in ('norm', 'stem', 'split', 'memset'))
    line = {'gpu': gpu_info(), 'shape': {'B': B, 'H': H, 'W': W}, 'ms_per_call': ms,
            'kernel_ms_by_kind': kinds, 'serial_hbm_pass_ms': round(hbm, 4),
            'concurrent_vs_serial_graph': round(ms['serial']['median'] / ms['concurrent']['median'], 4),
            'timing': f'CUDA graph replays, {args.reps} per window, median / best of {args.repeats} windows; kernel kinds '
                      'from a separate torch.profiler run of 5 eager calls'}
    text = json.dumps(line)
    print(text)
    with open(os.path.join(args.out, 'bench_encode.json'), 'w') as f:
        f.write(text + '\n')


if __name__ == '__main__':
    main()
