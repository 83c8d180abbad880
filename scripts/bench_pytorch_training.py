"""The cost of training under RAFT(conventions='pytorch') against the default conventions, on one GPU.

    python scripts/bench_pytorch_training.py [--rounds 5] [--calls 200] [--steps 4] [--out DIR]

  * lookup backward: CUDA-event ms per raft_b200_corr_lookup_backward_ex call, RAFT_SAMPLER_GRID (d/d pyramid only)
    against RAFT_SAMPLER_TF (d/d pyramid and d/d coords), the two alternating, at the Chairs shape (B = 4, 46 x 62) and a
    Sintel fine-tune shape (B = 6, 46 x 96), r = 4, 4 levels; coordinates are the query grid plus a smooth flow;
  * train_step: pairs/s of RAFT at the Chairs config (batch 4, 368 x 496, 12 iterations) with conventions 'pytorch'
    (TorchAdamW + OneCycleLR) against 'tf-raft' (AdamW), train precision fp32 and f16x2, the conventions alternating
    within each precision, `--steps` synchronised steps per round after two warm-up steps.
Medians over the rounds, with the card's name and power limit read in the same run.  One JSON line on stdout, and
DIR/bench_pytorch_training.json with --out."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), '..')))

import tf_raft_b200 as T  # noqa: E402
from tf_raft_b200 import _lib  # noqa: E402

LOOKUP_SHAPES = {'chairs': (4, 46, 62), 'sintel': (6, 46, 96)}
LEVELS, RADIUS = 4, 4


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else 'unknown'


def lookup_case(b, h, w, seed=0):
    rng = np.random.default_rng(seed)
    gy, gx = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing='ij')
    fx = 6 * np.sin(gy / 9 + 0.3) + 3 * np.cos(gx / 13) + rng.normal(0, 0.4, (b, h, w))
    fy = 4 * np.cos(gx / 11 - 0.2) - 2 * np.sin(gy / 7) + rng.normal(0, 0.4, (b, h, w))
    coords = torch.from_numpy(np.stack([gx + fx, gy + fy], axis=-1).astype(np.float32)).cuda()
    gen = torch.Generator(device='cuda').manual_seed(seed)
    pyr = [torch.randn((b * h * w, h >> l, w >> l), generator=gen, device='cuda') for l in range(LEVELS)]
    go = torch.randn((b, h, w, LEVELS * (2 * RADIUS + 1) ** 2), generator=gen, device='cuda') * 1e-3
    gpyr = [torch.zeros_like(p) for p in pyr]
    gc = torch.zeros_like(coords)
    return pyr, coords, go, gpyr, gc


def time_lookup(case, sampler, calls):
    pyr, coords, go, gpyr, gc = case
    b, h, w, _ = coords.shape
    args = (_lib.ptr_array(pyr), _lib.ptr(coords), _lib.ptr(go), b, h, w, LEVELS, RADIUS,
            _lib.ptr(gc if sampler == 'tf-raft' else None), _lib.ptr_array(gpyr), _lib.SAMPLERS[sampler])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        _lib.call('corr_lookup_backward_ex', coords.device, *args)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def train_model(conventions, train_precision):
    model = T.RAFT(iters=12, iters_pred=12, precision='f16x2', conventions=conventions)
    if conventions == 'pytorch':
        from oracle import raft_pytorch as rp
        model.load_pytorch_weights(rp.synthetic_checkpoint(seed=0))
        opt = T.TorchAdamW(weight_decay=1e-4, learning_rate=T.OneCycleLR(4e-4, 100100))
    else:
        opt = T.AdamW(weight_decay=1e-4, learning_rate=4e-4)
    model.compile(optimizer=opt, clip_norm=1.0, train_precision=train_precision)
    return model


def time_steps(model, batch, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        model.train_step(batch)
    torch.cuda.synchronize()
    return steps * batch[0].shape[0] / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--calls', type=int, default=200)
    ap.add_argument('--steps', type=int, default=4)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_pytorch_training needs a CUDA device')
    res = {'card': card(), 'lookup_backward_ms': {}, 'train_step_pairs_per_s': {}}
    for name, (b, h, w) in LOOKUP_SHAPES.items():
        case = lookup_case(b, h, w)
        for s in ('grid_sample', 'tf-raft'):                                    # warm-up
            time_lookup(case, s, 5)
        ms = {'grid_sample': [], 'tf-raft': []}
        for _ in range(args.rounds):
            for s in ms:
                ms[s].append(time_lookup(case, s, args.calls))
        res['lookup_backward_ms'][name] = {'B': b, 'h': h, 'w': w,
                                           **{s: round(statistics.median(v), 4) for s, v in ms.items()}}
        del case
    rng = np.random.default_rng(0)
    b, H, W = 4, 368, 496
    batch = (torch.from_numpy(rng.uniform(0, 255, (b, H, W, 3)).astype(np.float32)).cuda(),
             torch.from_numpy(rng.uniform(0, 255, (b, H, W, 3)).astype(np.float32)).cuda(),
             torch.from_numpy((rng.standard_normal((b, H, W, 2)) * 5).astype(np.float32)).cuda(),
             torch.from_numpy(rng.uniform(size=(b, H, W)) > 0.1).cuda())
    for tp in ('fp32', 'f16x2'):
        models = {c: train_model(c, tp) for c in ('pytorch', 'tf-raft')}
        for m in models.values():
            time_steps(m, batch, 2)                                              # warm-up
        rates = {c: [] for c in models}
        for _ in range(max(1, args.rounds // 2)):
            for c, m in models.items():
                rates[c].append(time_steps(m, batch, args.steps))
        res['train_step_pairs_per_s'][tp] = {c: round(statistics.median(v), 2) for c, v in rates.items()}
        del models
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_pytorch_training.json'), 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
