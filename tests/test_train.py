"""Training step (tf_raft/model.py:126-144) against torch.autograd of the CPU oracle.

CPU part: learning-rate schedule and optimiser arithmetic known answers.  GPU part: lookup backward vs autograd of the
oracle sampler, one full train_step (loss, clipped AdamW update of every variable) vs the same step done with
torch.autograd on the oracle forward.
"""
import math

import numpy as np
import pytest
import torch

import cases
from oracle import raft_torch as rt, weights


# --------------------------------------------------------------------------------------------- CPU
def test_cyclical_learning_rate_known_answers():
    """tfa CyclicalLearningRate(scale_mode='cycle') with first_cycle_scaler (train_chairs.py:79-85, training.py:10-15):
    min -> max over step_size steps, back to min over the next step_size, then constant min."""
    from tf_raft_b200.train import CyclicalLearningRate, first_cycle_scaler, inverse_scaler
    lr = CyclicalLearningRate(1e-4, 2e-4, 1000, scale_fn=first_cycle_scaler)
    assert lr(0) == pytest.approx(1e-4)
    assert lr(500) == pytest.approx(1.5e-4)
    assert lr(1000) == pytest.approx(2e-4)
    assert lr(1500) == pytest.approx(1.5e-4)
    assert lr(2000) == pytest.approx(1e-4)
    assert lr(2500) == pytest.approx(1e-4) and lr(3000) == pytest.approx(1e-4)      # cycle 2: scale 0
    inv = CyclicalLearningRate(1e-4, 2e-4, 1000, scale_fn=inverse_scaler)
    assert inv(3000) == pytest.approx(1e-4 + 1e-4 / 2)                               # peak of cycle 2, scaled 1/2
    assert first_cycle_scaler(1) == 1.0 and first_cycle_scaler(2) == 0.0


class _CpuLookup:
    """CPU stand-in for the CUDA lookup function: the oracle sampler under autograd."""
    @staticmethod
    def apply(coords, radius, *pyr):
        cb = rt.CorrBlock.__new__(rt.CorrBlock)
        cb.corr_pyramid, cb.num_levels, cb.radius = list(pyr), len(pyr), radius
        return cb.retrieve(coords)


class _CpuCorrBlock:
    def __init__(self, f1, f2, num_levels=4, radius=4, precision=None):
        self.corr_pyramid = [p.contiguous() for p in rt.CorrBlock(f1, f2, num_levels, radius).corr_pyramid]


@pytest.mark.parametrize('variant,iters', [('small', 3), ('raft', 2)])
def test_train_graph_and_corr_backward_match_oracle_autograd_on_cpu(monkeypatch, variant, iters):
    """Host logic of the training step without a GPU: the backward-capable graph (tf_raft_b200/train.py) with the two
    CUDA-backed autograd functions replaced by CPU stand-ins -- the lookup by the oracle sampler, the correlation FORWARD by
    the oracle volume while its hand-derived BACKWARD (GEMMs on pooled features) stays -- must give the oracle's loss and
    the oracle's torch.autograd gradient for every trainable variable."""
    import tf_raft_b200.train as tr
    from tf_raft_b200.losses import sequence_loss
    monkeypatch.setattr(tr, '_Lookup', _CpuLookup)
    monkeypatch.setattr(tr, 'CorrBlock', _CpuCorrBlock)
    p = weights.init_params(variant, 21, bias_scale=0.05, norm_jitter=0.1)
    im1, im2 = cases.images(2, 64, 96, 3, 4)
    rng = np.random.default_rng(9)
    flow_gt = torch.from_numpy((rng.standard_normal((2, 64, 96, 2)) * 5).astype(np.float32))
    valid = torch.from_numpy(rng.uniform(size=(2, 64, 96)) > 0.1)
    frozen = ('moving_mean', 'moving_variance')
    leaves = {k: torch.tensor(v, dtype=torch.float32, requires_grad=not k.endswith(frozen)) for k, v in p.items()}
    names = [k for k, v in leaves.items() if v.requires_grad]
    loss_o = sequence_loss([flow_gt, valid], rt.forward(leaves, im1, im2, variant, iters, training=True))
    g_o = dict(zip(names, torch.autograd.grad(loss_o, [leaves[k] for k in names])))
    P = {k: torch.tensor(v, dtype=torch.float32, requires_grad=not k.endswith(frozen)) for k, v in p.items()}
    moving = {k: v.detach().clone() for k, v in P.items() if k.endswith(frozen)}
    graph = tr.TrainGraph(P, variant, 'fp32', moving)
    loss = sequence_loss([flow_gt, valid], graph.forward(torch.from_numpy(im1), torch.from_numpy(im2), iters))
    assert float(loss) == pytest.approx(float(loss_o), rel=1e-5)
    g_t = dict(zip(names, torch.autograd.grad(loss, [P[k] for k in names])))
    for k in names:
        tol = 1e-4 * float(g_o[k].abs().max()) + 2e-6
        assert float((g_t[k] - g_o[k]).abs().max()) <= tol, k
    if variant == 'raft':        # keras BatchNormalization: moving statistics move by (1 - 0.99) of the batch statistics
        assert any(float((moving[k] - P[k]).abs().max()) > 0 for k in moving)


# --------------------------------------------------------------------------------------------- GPU
gpu = pytest.mark.gpu


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@gpu
def test_lookup_backward_vs_oracle_autograd():
    """d/d coords and d/d pyramid of CorrBlock.retrieve: the CUDA kernel against torch.autograd of the oracle sampler
    (floor / ceil / gather carry no gradient, clamp passes it inside the range -- TensorFlow's rules)."""
    from tf_raft_b200.train import _Lookup
    b, h, w, c, r, levels = 2, 8, 12, 64, 4, 4
    f1, f2 = cases.fmaps(b, h, w, c)
    ocb = rt.CorrBlock(torch.from_numpy(f1), torch.from_numpy(f2), levels, r)
    coords_np = cases.lookup_coords(b, h, w, 'jitter')
    pyr_cpu = [p.clone().requires_grad_(True) for p in ocb.corr_pyramid]
    ocb.corr_pyramid = pyr_cpu
    coords_cpu = torch.from_numpy(coords_np).requires_grad_(True)
    out_cpu = ocb.retrieve(coords_cpu)
    g = torch.from_numpy(np.random.default_rng(5).standard_normal(tuple(out_cpu.shape)).astype(np.float32))
    out_cpu.backward(g)
    pyr_gpu = [p.detach().cuda().requires_grad_(True) for p in pyr_cpu]
    coords_gpu = dev(coords_np).requires_grad_(True)
    out_gpu = _Lookup.apply(coords_gpu, r, *pyr_gpu)
    np.testing.assert_array_equal(out_gpu.detach().cpu().numpy(), out_cpu.detach().numpy())
    out_gpu.backward(g.cuda())
    np.testing.assert_allclose(coords_gpu.grad.cpu().numpy(), coords_cpu.grad.numpy(), atol=2e-4, rtol=1e-4)
    for l in range(levels):
        np.testing.assert_allclose(pyr_gpu[l].grad.cpu().numpy(), pyr_cpu[l].grad.numpy(), atol=1e-5, rtol=1e-5, err_msg=f'level {l}')


def _oracle_step(params, im1, im2, flow_gt, valid, variant, iters, clip_norm, lr, wd, beta1=0.9, beta2=0.999, eps=1e-7):
    """One training step with torch.autograd on the CPU oracle: loss, clipped gradients, AdamW update (t = 1)."""
    leaves = {k: torch.tensor(v, dtype=torch.float32, requires_grad=not k.endswith(('moving_mean', 'moving_variance')))
              for k, v in params.items()}
    preds = rt.forward(leaves, im1, im2, variant, iters, training=True)
    fg = torch.from_numpy(flow_gt)
    va = torch.from_numpy(valid)
    mag = torch.sqrt((fg ** 2).sum(-1))
    vm = (va & (mag < 400)).float().unsqueeze(-1)
    loss = sum(0.8 ** (iters - i - 1) * (vm * (p - fg).abs()).mean() for i, p in enumerate(preds))
    names = [k for k, v in leaves.items() if v.requires_grad]
    grads = torch.autograd.grad(loss, [leaves[k] for k in names])
    norm = math.sqrt(sum(float((g.double() ** 2).sum()) for g in grads))
    scale = clip_norm / max(norm, clip_norm)
    new = {}
    lr_t = lr * math.sqrt(1 - beta2) / (1 - beta1)
    for k, g in zip(names, grads):
        g = g * scale
        w = leaves[k].detach()
        w = w - wd * w
        m = (1 - beta1) * g
        v = (1 - beta2) * g * g
        new[k] = w - lr_t * m / (v.sqrt() + eps)
    return float(loss), norm, new, dict(zip(names, grads))


@gpu
@pytest.mark.parametrize('variant,shape,iters', [('small', (64, 96), 3), ('raft', (64, 96), 2)])
def test_train_step_vs_oracle_autograd(variant, shape, iters):
    """RAFT.train_step = the reference's train_step (model.py:126-144): same loss, same global gradient norm, and the
    updated value of EVERY trainable variable within 1e-4 relative of an oracle torch.autograd step."""
    import tf_raft_b200 as T
    from tf_raft_b200.train import AdamW
    H, W = shape
    bsz = 2
    p = weights.init_params(variant, 21, bias_scale=0.05, norm_jitter=0.1)
    im1, im2 = cases.images(bsz, H, W, 3, 4)
    rng = np.random.default_rng(9)
    flow_gt = (rng.standard_normal((bsz, H, W, 2)) * 5).astype(np.float32)
    valid = rng.uniform(size=(bsz, H, W)) > 0.1
    clip_norm, lr, wd = 1.0, 1e-4, 1e-5
    loss_o, norm_o, new_o, grads_o = _oracle_step(p, im1, im2, flow_gt, valid, variant, iters, clip_norm, lr, wd)
    cls = T.RAFT if variant == 'raft' else T.SmallRAFT
    model = cls(iters=iters, iters_pred=iters, precision='f16x2')
    model.load_params(p)
    model.compile(optimizer=AdamW(weight_decay=wd, learning_rate=lr), clip_norm=clip_norm)
    out = model.train_step((dev(im1), dev(im2), dev(flow_gt), torch.from_numpy(valid).cuda()))
    assert out['loss'] == pytest.approx(loss_o, rel=2e-4), (out['loss'], loss_o)
    # gradients of every trainable variable (the flat gradient buffer still holds the unclipped, all-reduced gradients)
    tr = model._trainer
    gnorm = math.sqrt(float((tr.flat.g.double() ** 2).sum()))
    assert gnorm == pytest.approx(norm_o, rel=1e-3), (gnorm, norm_o)
    # Per variable and globally.  The two sides differ in arithmetic (tensor-core fp16 hi/lo correlation and PyTorch CUDA convolutions vs
    # CPU fp32, atomics in the lookup scatter) and the loss is only piecewise smooth in the coordinates (floor / ceil sampler),
    # so individual entries agree to a fraction of a percent of the tensor's scale, the whole gradient to 1e-2 in norm.
    num = den = 0.0
    for k, want in grads_o.items():
        got_g = tr.flat.views[k].grad.cpu()
        num += float(((got_g - want).double() ** 2).sum())
        den += float((want.double() ** 2).sum())
        tol = 5e-2 * float(want.abs().max()) + 2e-6       # (biases in front of a norm layer have a zero true gradient: noise)
        assert float((got_g - want).abs().max()) <= tol, f'gradient of {k}: max error {float((got_g - want).abs().max()):.3e} (scale {float(want.abs().max()):.3e})'
    assert math.sqrt(num / den) <= 1e-2, f'relative L2 error of the whole gradient {math.sqrt(num / den):.3e}'
    # updated values.  Adam's first step is lr * g / (|g| + eps'): a sign-like function of the gradient, so an entry whose
    # gradient is small relative to the tensor's (and, after clipping, to Adam's epsilon / sqrt(1 - beta2) = 3e-6) is decided
    # by rounding; the comparison is made where the gradient is well-determined (|g| >= 20 % of the tensor's largest), on
    # the UPDATE (new - old), to 5 % of the learning rate.
    got = {k: v.cpu() for k, v in model.state_dict().items()}
    worst = 0.0
    for k, want in new_o.items():
        g = grads_o[k]
        sel = g.abs() >= 0.2 * g.abs().max()
        if float(g.abs().max()) < 1e-5 or not bool(sel.any()):          # zero true gradient: noise
            continue
        old = torch.from_numpy(np.asarray(p[k], dtype=np.float32))
        err = float(((got[k] - old) - (want - old))[sel].abs().max()) / lr
        worst = max(worst, err)
        assert err <= 5e-2, f'{k}: update differs by {err:.3f} x lr (global norm oracle {norm_o:.4f})'
    print(f'{variant}: loss {out["loss"]:.6f} (oracle {loss_o:.6f}), worst update error {worst:.3f} x lr')
