"""Self-supervised against supervised training steps at the Chairs config, and the loss kernels' share of a step.

    python scripts/bench_unsup.py [--out DIR] [--rounds 5 --steps 3 --warmup 3]

RAFT, batch 4, 368x496, 12 iterations (train_chairs.yml), AdamW, clip 1.0, on seeded synthetic pairs resident on the
device.  Two models from the same weights: one compiled with the default sequence loss, one with UnsupervisedLoss.
Their `train_step`s alternate in `--rounds` rounds of `--steps` steps, each round timed with a host clock that ends in a
device synchronise; pairs/s per round, the median, and the ratio of the medians are reported.  The unsupervised step
runs the update loop at batch 2B (both directions), so it is expected to be slower; the script measures by how much.

Loss kernels per step, CUDA events over 20 calls on predictions of the step's shapes (2 x 12 x (4, 368, 496, 2)):
the census of the 2B images (raft_b200_census), the two loss-and-gradient calls (raft_b200_unsup_loss, three kernels
each), and the whole UnsupervisedLoss forward and backward (occlusion check, census, stacking, loss, gradient scale).
The GPU's name, power limit and maximum SM clock are read (nvidia-smi, query only) in the same run: one JSON line on
stdout, and in DIR/bench_unsup.json with --out.
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

import tf_raft_b200 as T  # noqa: E402
from tf_raft_b200.losses import census_transform  # noqa: E402
from tf_raft_b200.train import AdamW, _UnsupLoss  # noqa: E402

BATCH, H, W, ITERS = 4, 368, 496, 12


def gpu_info():
    try:
        res = subprocess.run(['nvidia-smi', f'--id={torch.cuda.current_device()}',
                              '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=60)
        return res.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f'nvidia-smi unavailable: {e}'


def batch(seed):
    """A textured image and its copy moved by (3, 1) px, with that flow as ground truth."""
    rng = np.random.default_rng(seed)
    small = rng.uniform(0, 255, (BATCH, H // 4, W // 4, 3)).astype(np.float32)
    im1 = torch.from_numpy(np.repeat(np.repeat(small, 4, axis=1), 4, axis=2)).cuda()
    im2 = torch.roll(im1, shifts=(1, 3), dims=(1, 2))
    flow = torch.zeros((BATCH, H, W, 2), device='cuda')
    flow[..., 0], flow[..., 1] = 3.0, 1.0
    return im1, im2, flow, torch.ones((BATCH, H, W), device='cuda')


def event_ms(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps


def loss_kernels(data, reps=20):
    im1, im2 = data[0], data[1]
    rng = torch.Generator(device='cuda').manual_seed(0)
    preds = [[(torch.randn((BATCH, H, W, 2), device='cuda', generator=rng) * 3).requires_grad_(True)
              for _ in range(ITERS)] for _ in range(2)]
    loss_fn = T.UnsupervisedLoss()
    images = torch.cat([im1, im2]).contiguous()
    census = census_transform(images)
    occ = torch.cat(T.fb_occlusion(preds[0][-1].detach(), preds[1][-1].detach()))
    flows = torch.stack([p.detach() for p in preds[0] + preds[1]])
    args = (loss_fn.census_weight, loss_fn.smoothness_weight, loss_fn.edge_weight, loss_fn.gamma)

    def whole():
        loss = loss_fn((im1, im2), preds)
        torch.autograd.grad(loss, preds[0] + preds[1])

    return {'census_ms': event_ms(lambda: census_transform(images), reps),
            'loss_and_gradient_ms': event_ms(lambda: _UnsupLoss.apply(flows, census, images, occ, *args), reps),
            'unsupervised_loss_forward_backward_ms': event_ms(whole, reps)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--out', default=None)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_unsup.py measures on the GPU; no CUDA device found')
    torch.cuda.set_device(0)
    data = batch(0)
    models = {}
    for name, loss in (('supervised', T.sequence_loss), ('unsupervised', T.UnsupervisedLoss())):
        model = T.RAFT(iters=ITERS, iters_pred=ITERS, seed=0)
        model.compile(optimizer=AdamW(weight_decay=1e-4, learning_rate=1e-4), clip_norm=1.0, loss=loss)
        models[name] = model
    step_data = {'supervised': data, 'unsupervised': data[:2]}
    for name, model in models.items():
        for _ in range(args.warmup):
            model.train_step(step_data[name])
    torch.cuda.synchronize()
    rates = {name: [] for name in models}
    for _ in range(args.rounds):
        for name, model in models.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                out = model.train_step(step_data[name])
            torch.cuda.synchronize()
            rates[name].append(BATCH * args.steps / (time.perf_counter() - t0))
            assert np.isfinite(out['loss'])
    med = {name: statistics.median(r) for name, r in rates.items()}
    result = {'config': f'RAFT batch {BATCH} {H}x{W} iters {ITERS}', 'gpu': gpu_info(),
              'supervised_pairs_per_s': round(med['supervised'], 2),
              'unsupervised_pairs_per_s': round(med['unsupervised'], 2),
              'unsupervised_over_supervised': round(med['unsupervised'] / med['supervised'], 3),
              'rounds': {k: [round(v, 2) for v in r] for k, r in rates.items()},
              'peak_memory_gb': round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}
    result.update({k: round(v, 3) for k, v in loss_kernels(data).items()})
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_unsup.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
