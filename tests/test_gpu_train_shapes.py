"""The training step at the shapes it is trained at, against a teacher-forced float64 gradient.

Every other end-to-end training test runs at 64x96 with 2 or 3 iterations.  Here one `RAFT.train_step` runs at the
FlyingChairs configuration (batch 4, 368x496 crops, 12 iterations; RAFT, SmallRAFT and RAFT(conventions='pytorch')) and
at a KITTI one (batch 2, 288x960, sparse ground truth with a band beyond the 400 px magnitude mask), each with
train_precision 'fp32' and 'f16x2', and is compared with the same step in float64 on the GPU: oracle.raft_torch
(tf-raft) or tests/pytorch_train_oracle.py (pytorch) under torch.autograd, teacher-forced by oracle/teacher_forced.py
-- every lookup samples at the GPU's own float32 positions, while the gradient flows through the reference's own
float64 coordinates.  That makes the comparison well conditioned over all twelve links of tf-raft's
coordinate-gradient chain, so the gates below are set from measurement.

Compared, each as a ratio: the loss (relative); every prediction (max-abs error over the prediction's max-abs); the
global gradient norm (relative); the whole gradient (relative L2); every gradient tensor by relative L2 and by max-abs
error over its max-abs, the worst tensor of fnet, cnet and the update block reported; the conv biases in front of a
normalisation, whose exact gradient is 0 (max-abs over the largest gradient entry of the model); under 'tf-raft', d loss
/ d coords1 of every iteration (relative L2; an iteration the gradient does not reach counts as 1); and, for RAFT,
cnet's moving statistics (max-abs error over the largest change the step made).  The parameter update is not compared:
Adam's first step is sign-like, and the optimiser has its own fp64 tests.

Each gate is 3x the worst ratio measured on the unmodified code over three seeds.  These faults each exceed a gate of
every case they can reach: the coarsest level left out of d fmap1 or the 1/sqrt(C) scale dropped on the d fmap2 branch
(fnet and whole-gradient L2, >= 9x their gates), levels >= 2 left out of the lookup's coordinate gradient or coords1
detached at the top of each tf-raft iteration (coords_grad, >= 20x), and, under 'f16x2', the last slice of the tensor
cores' weight-gradient reduction left out (norm, > 1000x).  A coordinate gradient scaled by 1 - 2^-7 exceeds the
coords_grad gate by only 1.9-2.9x: the fp32 chain of twelve iterations carries up to 6.5e-4 relative error by itself.
The coordinate faults cannot act under conventions='pytorch', whose lookup has no coordinate gradient.
"""
import contextlib
import math
import re
import time
from unittest import mock

import numpy as np
import pytest
import torch

import cases
import pytorch_train_oracle as pto
from oracle import raft_pytorch as rp, teacher_forced as tfo, train_ref, weights

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, torch.float64
ITERS = 12
CLIP = 1.0                        # below the gradient norm of every case (asserted): the clip acts

CASES = {
    'chairs': dict(variant='raft', conventions='tf-raft', b=4, H=368, W=496, data='chairs'),
    'chairs-small': dict(variant='small', conventions='tf-raft', b=4, H=368, W=496, data='chairs'),
    'kitti': dict(variant='raft', conventions='tf-raft', b=2, H=288, W=960, data='kitti'),
    'chairs-pytorch': dict(variant='raft', conventions='pytorch', b=4, H=368, W=496, data='chairs'),
}

PARTS = ('fnet', 'cnet', 'update_block')          # gradient tensors are reported per part of the model

# Gates on the ratios of compare(), per train_precision: 3x the worst ratio measured on an H100 SXM (700 W) over seeds
# 0, 1, 2 and the four cases, rounded up.  The encoders' per-tensor ratios (fnet_*, cnet_*) are large because the fp32
# step's conv kernel gradients in front of a normalisation cancel heavily (up to 2.7e-2 max-abs measured); their L2 and
# the whole-gradient L2 are what catch faults there.
GATES = {
    'fp32': dict(loss=8e-7, preds=2e-5, norm=2e-5, grad_l2=2e-4, fnet_l2=2e-2, fnet_max=8e-2, cnet_l2=2e-2,
                 cnet_max=9e-2, update_block_l2=6e-4, update_block_max=3e-3, zero_grad=1e-7, coords_grad=2e-3,
                 moving=2e-4),
    'f16x2': dict(loss=2e-5, preds=2e-5, norm=2e-5, grad_l2=2e-4, fnet_l2=2e-2, fnet_max=8e-2, cnet_l2=2e-2,
                  cnet_max=7e-2, update_block_l2=1e-3, update_block_max=7e-3, zero_grad=2e-7, coords_grad=2e-3,
                  moving=2e-4),
}


@pytest.fixture(scope='module')
def T():
    import tf_raft_b200
    from tf_raft_b200 import _lib
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    return tf_raft_b200


# --------------------------------------------------------------------------------------------- workloads
def batch(case, seed):
    """Images (uniform 0..255), ground truth and valid mask of a case.  'chairs': dense valid, a smooth flow of a few px
    plus sub-pixel detail; 'kitti': ~25 % valid, and a band of rows whose ground truth exceeds 400 px, which the
    magnitude mask must drop."""
    c = CASES[case]
    b, H, W = c['b'], c['H'], c['W']
    im1, im2 = cases.images(b, H, W, 100 + seed, 200 + seed)
    rng = np.random.default_rng(300 + seed)
    y, x = np.meshgrid(np.arange(H), np.arange(W), indexing='ij')
    flow = np.empty((b, H, W, 2))
    for i in range(b):
        for ch in range(2):
            fy, fx, ph = rng.uniform(0.5, 3, 3)
            flow[i, :, :, ch] = 3 * np.sin(2 * np.pi * (fy * y / H + fx * x / W) + 6 * ph)
    flow += 0.3 * rng.standard_normal(flow.shape)
    if c['data'] == 'chairs':
        valid = np.ones((b, H, W), bool)
    else:
        valid = rng.uniform(size=(b, H, W)) < 0.25
        band = slice(H // 3, H // 3 + 24)
        flow[:, band, :, 0] = 400 + 100 * rng.uniform(size=(b, 24, W))
        valid[:, band] = True
    return im1, im2, flow.astype(F32), valid


def is_structural_zero(name, case):
    """A conv bias in front of a normalisation layer: its exact gradient is 0 (instance norm in fnet, batch norm in
    RAFT's cnet; SmallRAFT's cnet has no norm)."""
    enc = re.fullmatch(r'(fnet|cnet)\.(conv1|layer\d\.\d\.(conv1|conv2|downsample\.0))\.bias', name)
    return bool(enc) and not (enc.group(1) == 'cnet' and CASES[case]['variant'] == 'small')


# --------------------------------------------------------------------------------------------- the GPU step
def watch_coords_grad(coords, k, store):
    """Keeps d loss / d coords1 of iteration k (all its uses: the lookup, the flow input, the next coords1) in
    store[k]."""
    if coords.requires_grad:
        coords.register_hook(lambda g: store.__setitem__(k, g.detach().double().cpu()))


@contextlib.contextmanager
def recording():
    """Keeps the float32 coordinates each iteration's lookup receives and the step's predictions."""
    import tf_raft_b200.train as tr
    rec = dict(coords=[], preds=[], coords_grad={})

    def recorder(fn):
        class Recorded:
            @staticmethod
            def apply(coords, radius, *pyramid):
                watch_coords_grad(coords, len(rec['coords']), rec['coords_grad'])
                rec['coords'].append(coords.detach().clone())
                return fn.apply(coords, radius, *pyramid)
        return Recorded

    iterate = tr.TrainGraph._iterate

    def _iterate(self, *args, **kwargs):
        preds = iterate(self, *args, **kwargs)
        rec['preds'] = [p.detach() for p in preds]
        return preds

    with mock.patch.object(tr, '_Lookup', recorder(tr._Lookup)), \
            mock.patch.object(tr, '_GridLookup', recorder(tr._GridLookup)), \
            mock.patch.object(tr.TrainGraph, '_iterate', _iterate):
        yield rec


def model_for(T, case, seed, train_precision):
    """A fresh model of the case with seeded weights, compiled for one train_step; also the weights (project names for
    tf-raft, the PyTorch-layout checkpoint for conventions='pytorch')."""
    c = CASES[case]
    if c['conventions'] == 'pytorch':
        ckpt = rp.synthetic_checkpoint(seed=seed)
        m = T.RAFT(conventions='pytorch', precision='f16x2', device='cuda', iters=ITERS, iters_pred=ITERS)
        m.load_pytorch_weights(ckpt)
        m.compile(optimizer=T.TorchAdamW(weight_decay=1e-4, learning_rate=1e-4), clip_norm=CLIP,
                  train_precision=train_precision)
        return m, ckpt
    from tf_raft_b200.train import AdamW
    p = weights.init_params(c['variant'], seed, bias_scale=0.05, norm_jitter=0.1)
    m = (T.RAFT if c['variant'] == 'raft' else T.SmallRAFT)(iters=ITERS, iters_pred=ITERS, precision='f16x2')
    m.load_params(p)
    m.compile(optimizer=AdamW(weight_decay=1e-4, learning_rate=1e-4), clip_norm=CLIP, train_precision=train_precision)
    return m, p


def gpu_step(T, case, seed, train_precision, data):
    """One train_step; returns dict(loss, preds, grads {project name: float64 CPU tensor}, moving, coords, weights)."""
    model, w = model_for(T, case, seed, train_precision)
    im1, im2, flow, valid = data
    with recording() as rec:
        out = model.train_step((torch.from_numpy(im1).cuda(), torch.from_numpy(im2).cuda(),
                                torch.from_numpy(flow).cuda(), torch.from_numpy(valid).cuda()))
    tr = model._trainer
    assert len(rec['coords']) == len(rec['preds']) == ITERS
    return dict(loss=float(out['loss']), preds=rec['preds'], coords=rec['coords'], weights=w,
                coords_grad=rec['coords_grad'],
                grads={k: v.grad.detach().double().cpu() for k, v in tr.flat.views.items()},
                moving={k: v.detach().double().cpu() for k, v in tr.moving.items()})


# --------------------------------------------------------------------------------------------- the fp64 reference
def _to_project(T, grads):
    """{PyTorch name: tensor} -> {project name: float32 ndarray} (fnet norms excluded), as test_gpu_pytorch_training
    maps them.  The float32 rounding of the reference (6e-8 relative) is far below every gate."""
    sd = {k: v.detach().cpu().float().numpy() for k, v in grads.items()}
    for k in list(sd):
        if '.downsample.1.' in k:
            sd[k.replace('.downsample.1.', '.norm3.')] = sd[k]
    out = T.load_pytorch_checkpoint(sd)
    return {k: v for k, v in out.items() if not (k.startswith('fnet.') and k.endswith(('.gamma', '.beta')))}


def reference(T, case, weights_, data, coords, device='cuda'):
    """The float64 step on the GPU, teacher-forced by the recorded coordinates: dict(loss, preds, grads {project name:
    float64 CPU tensor}, moving {name: float64 CPU tensor}, moving0)."""
    c = CASES[case]
    im1, im2, flow, valid = data
    if c['conventions'] == 'pytorch':
        sd = {k: v.to(device, F64).requires_grad_(pto.trainable(k)) for k, v in rp._sd(weights_, F64).items()}
        names = [k for k in sd if pto.trainable(k)]
        moving0 = _to_project(T, {k: v.detach().clone() for k, v in sd.items() if 'running' in k})

        def lookup(k, pyr, coords1):
            return tfo.grid_lookup(pyr, coords[k].permute(0, 3, 1, 2))
        preds = pto.train_forward(sd, im1, im2, ITERS, 'train', F64, lookup=lookup)
        loss = pto.sequence_loss(preds, torch.from_numpy(flow), torch.from_numpy(valid))
        g = torch.autograd.grad(loss, [sd[k] for k in names])
        grads = {k: torch.from_numpy(v).double() for k, v in _to_project(T, dict(zip(names, g))).items()}
        moving = {k: torch.from_numpy(v).double() for k, v in
                  _to_project(T, {k: v.detach() for k, v in sd.items() if 'running' in k}).items()
                  if k.endswith(tfo.FROZEN)}
        moving0 = {k: torch.from_numpy(v).double() for k, v in moving0.items() if k.endswith(tfo.FROZEN)}
        return dict(loss=float(loss), preds=[p.detach() for p in preds], grads=grads, moving=moving, moving0=moving0)
    coords_grad, retrieve = {}, tfo.tf_retrieve

    def watched(corr_block, c64, c32):
        watch_coords_grad(c64, len(coords_grad_calls), coords_grad)
        coords_grad_calls.append(None)
        return retrieve(corr_block, c64, c32)
    coords_grad_calls = []
    with mock.patch.object(tfo, 'tf_retrieve', watched):
        loss, preds, grads, rec = tfo.tf_step(weights_, im1, im2, flow, valid, c['variant'], coords, device=device)
    moving0 = {k: np.asarray(v, np.float64) for k, v in weights_.items() if k.endswith(tfo.FROZEN)}
    stats = {k: (m.cpu().numpy(), v.cpu().numpy(), n) for k, (m, v, n) in rec.items()}
    moving = train_ref.bn_moving_update(moving0, stats)
    return dict(loss=loss, preds=preds, grads={k: v.cpu() for k, v in grads.items()}, coords_grad=coords_grad,
                moving={k: torch.from_numpy(v) for k, v in moving.items()},
                moving0={k: torch.from_numpy(v) for k, v in moving0.items()})


# --------------------------------------------------------------------------------------------- comparison
def compare(case, got, want):
    """The ratios named in the module docstring, and the tensor each worst per-tensor ratio came from."""
    r, where = {}, {}
    r['loss'] = abs(got['loss'] - want['loss']) / abs(want['loss'])
    r['preds'] = max(float((g.double() - w.to(g.device)).abs().max() / w.abs().max())
                     for g, w in zip(got['preds'], want['preds']))
    assert sorted(got['grads']) == sorted(want['grads']), 'trainable sets differ'
    gn = math.sqrt(sum(float((g ** 2).sum()) for g in got['grads'].values()))
    wn = math.sqrt(sum(float((w ** 2).sum()) for w in want['grads'].values()))
    assert wn > CLIP, f'gradient norm {wn:.3f} must exceed the clip {CLIP}'
    r['norm'] = abs(gn - wn) / wn
    gmax = max(float(w.abs().max()) for w in want['grads'].values())
    num = den = 0.0
    r['zero_grad'] = 0.0
    for part in PARTS:
        r[part + '_l2'] = r[part + '_max'] = 0.0
    for k, w in want['grads'].items():
        e = got['grads'][k] - w
        if is_structural_zero(k, case):
            q = float(e.abs().max()) / gmax
            if q >= r['zero_grad']:
                r['zero_grad'], where['zero_grad'] = q, k
            continue
        num += float((e ** 2).sum())
        den += float((w ** 2).sum())
        part = k.split('.')[0]
        for key, q in ((part + '_l2', float(e.norm() / w.norm())),
                       (part + '_max', float(e.abs().max() / w.abs().max()))):
            if q >= r[key]:
                r[key], where[key] = q, k
    r['grad_l2'] = math.sqrt(num / den)
    if CASES[case]['conventions'] == 'tf-raft':          # the gradient through the twelve iterations of coords1
        assert sorted(want['coords_grad']) == list(range(1, ITERS))
        r['coords_grad'] = 0.0
        for k, w in want['coords_grad'].items():
            g = got['coords_grad'].get(k, torch.zeros_like(w))                 # none reached it: a broken chain
            q = float((g - w).norm() / w.norm())
            if q >= r['coords_grad']:
                r['coords_grad'], where['coords_grad'] = q, f'iteration {k + 1}'
    if CASES[case]['variant'] == 'raft':
        r['moving'] = 0.0
        for k, w in want['moving'].items():
            q = float((got['moving'][k] - w).abs().max() / (w - want['moving0'][k]).abs().max())
            if q >= r['moving']:
                r['moving'], where['moving'] = q, k
    return r, wn, where


def run_case(T, case, seed, train_precision):
    """GPU step, teacher-forced reference and their ratios; prints the cost of the case."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    data = batch(case, seed)
    got = gpu_step(T, case, seed, train_precision, data)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    want = reference(T, case, got['weights'], data, got['coords'])
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    ratios, norm, where = compare(case, got, want)
    print(f'{case} {train_precision} seed {seed}: GPU step {t1 - t0:.1f} s, fp64 reference {t2 - t1:.1f} s, '
          f'peak memory '
          f'{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB, loss {want["loss"]:.5f}, norm {norm:.3f}')
    return ratios, where, dict(data=data, want=want)


@pytest.mark.parametrize('train_precision', ['fp32', 'f16x2'])
@pytest.mark.parametrize('case', list(CASES))
def test_train_step_at_training_shape_vs_teacher_forced_fp64(T, case, train_precision):
    ratios, where, _ = run_case(T, case, 0, train_precision)
    gates = GATES[train_precision]
    print(f'{case} {train_precision}: worst ratio / gate: ' + ', '.join(
        f'{k} {v:.2e} / {gates[k]:.0e}' + (f' ({where[k]})' if k in where else '') for k, v in ratios.items()))
    bad = {k: v for k, v in ratios.items() if v > gates[k]}
    assert not bad, f'{case} {train_precision}: over the gate: {bad}'
