"""Training under RAFT(conventions='pytorch') on the GPU: the grid_sample lookup backward against its NumPy float32
emulation (bit for bit), the torch AdamW rule against the float64 torch optimiser, the training step against RAFT's
training forward restated in float64 with the real torch optimiser, determinism, the `.pth` export, a resumed fit and
the training script."""
import glob
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import cases
import pytorch_train_oracle as pto
from oracle import raft_pytorch as rp

pytestmark = pytest.mark.gpu
F32 = np.float32
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))


@pytest.fixture(scope='module')
def T():
    import tf_raft_b200
    from tf_raft_b200 import _lib
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    return tf_raft_b200


@pytest.fixture(scope='module')
def ckpt():
    return rp.synthetic_checkpoint(seed=11)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).cuda()


def same_bits(a, b):
    """Equal bit for bit, any NaN equal to any NaN."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and np.array_equal(a.view(np.uint32)[~nan],
                                                                                      b.view(np.uint32)[~nan])


# --------------------------------------------------------------------------------------------- 1. lookup backward
def _coords(b, h, w, kind):
    if kind in ('grid', 'jitter', 'edge'):
        return cases.lookup_coords(b, h, w, kind)
    c = cases.lookup_coords(b, h, w, 'jitter').reshape(-1, 2)
    rng = np.random.default_rng(4)
    specials = np.array([np.nan, np.inf, -np.inf, 1e30, -1e30, 0.0, w - 1.0, h - 1.0, -0.5, w - 0.5, -1.0, w + 0.25,
                         1e8, 2.0 ** 31, -(2.0 ** 31)], F32)
    pick = rng.integers(0, len(specials), c.shape)
    mask = rng.uniform(size=c.shape) < 0.5
    c[mask] = specials[pick[mask]]
    return c.reshape(b, h, w, 2).astype(F32)


def _backward(coords, go, gpyr_in, radius, sampler=1, pyr=None, grad_coords=None):
    from tf_raft_b200 import _lib
    b, h, w, _ = coords.shape
    g = [dev(x) for x in gpyr_in]
    p = [dev(x) for x in pyr] if pyr is not None else g
    c, o = dev(coords), dev(go)                            # held: the library reads them after this line
    _lib.call('corr_lookup_backward_ex', 'cuda', _lib.ptr_array(p), _lib.ptr(c), _lib.ptr(o), b, h, w, len(g), radius,
              _lib.ptr(grad_coords), _lib.ptr_array(g), sampler)
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in g]


def _inputs(b, h, w, levels, radius, kind, seed, specials=False):
    rng = np.random.default_rng(seed)
    coords = _coords(b, h, w, kind)
    go = rng.standard_normal((b, h, w, levels * (2 * radius + 1) ** 2)).astype(F32)
    gin = [rng.standard_normal((b * h * w, h >> l, w >> l)).astype(F32) for l in range(levels)]
    if specials:                                           # non-finite incoming gradients and accumulators
        flat = go.reshape(-1)
        idx = rng.choice(flat.size, max(1, flat.size // 50), replace=False)
        flat[idx] = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0], F32)[idx % 5]
        for g in gin:
            gf = g.reshape(-1)
            gf[rng.choice(gf.size, max(1, gf.size // 100), replace=False)] = np.nan
    return coords, go, gin


LOOKUP_CASES = [(lv, s) for lv, shapes in cases.LOOKUP_GRIDS.items() for s in shapes]


@pytest.mark.parametrize('levels,shape', LOOKUP_CASES)
@pytest.mark.parametrize('radius', [4, 3, 2])
@pytest.mark.parametrize('kind', ['grid', 'jitter', 'edge', 'special'])
def test_grid_lookup_backward_equals_emulation(T, levels, shape, radius, kind):
    b, h, w = shape
    coords, go, gin = _inputs(b, h, w, levels, radius, kind, levels * 31 + radius, specials=kind == 'special')
    want = pto.lookup_backward_emulated(coords, go, gin, radius)
    got = _backward(coords, go, gin, radius)
    for l in range(levels):
        assert same_bits(got[l], want[l]), f'level {l}: {np.flatnonzero(got[l] != want[l])[:5]}'
    again = _backward(coords, go, gin, radius)
    assert all(same_bits(a, g) for a, g in zip(again, got)), 'two calls differ'


@pytest.mark.parametrize('b,h,w', [(4, 46, 62), (6, 46, 96)], ids=['chairs', 'sintel'])
def test_grid_lookup_backward_at_training_shapes(T, b, h, w):
    coords, go, gin = _inputs(b, h, w, 4, 4, 'jitter', 5)
    coords = (coords + np.random.default_rng(6).standard_normal(coords.shape) * 6).astype(F32)
    want = pto.lookup_backward_emulated(coords, go, gin, 4)
    got = _backward(coords, go, gin, 4)
    for l in range(4):
        assert same_bits(got[l], want[l]), f'level {l}'
    assert all(same_bits(a, g) for a, g in zip(_backward(coords, go, gin, 4), got)), 'two calls differ'


def test_backward_ex_tf_sampler_and_argument_checks(T):
    from tf_raft_b200 import _lib
    b, h, w, levels, radius = 2, 9, 13, 4, 4
    coords, go, _ = _inputs(b, h, w, levels, radius, 'jitter', 8)
    f1, f2 = cases.fmaps(b, h, w, 32, 3)
    pyr = [p[:, 0].float().numpy() for p in rp.corr_pyramid(torch.from_numpy(f1).permute(0, 3, 1, 2).double(),
                                                             torch.from_numpy(f2).permute(0, 3, 1, 2).double(), levels)]
    outs = []
    dp, c, o = [dev(p) for p in pyr], dev(coords), dev(go)
    for fn in ('corr_lookup_backward', 'corr_lookup_backward_ex'):
        gc = torch.zeros((b, h, w, 2), device='cuda')
        gp = [torch.zeros(p.shape, device='cuda') for p in pyr]
        args = [_lib.ptr_array(dp), _lib.ptr(c), _lib.ptr(o), b, h, w, levels, radius, _lib.ptr(gc), _lib.ptr_array(gp)]
        _lib.call(fn, 'cuda', *(args + ([0] if fn.endswith('_ex') else [])))
        outs.append([gc.cpu().numpy()] + [x.cpu().numpy() for x in gp])
    assert all(same_bits(a, c) for a, c in zip(*outs))
    gc = torch.zeros((b, h, w, 2), device='cuda')
    gp = [torch.zeros(p.shape, device='cuda') for p in pyr]
    lib = _lib.lib()
    st = ctypes_stream()
    status = lib.raft_b200_corr_lookup_backward_ex(None, _lib.ptr(c), _lib.ptr(o), b, h, w, levels, radius,
                                                   _lib.ptr(gc), _lib.ptr_array(gp), 1, st)
    assert status == -1                                    # RAFT_ERR_BAD_ARG: the grid backward has no coordinate gradient
    assert lib.raft_b200_corr_lookup_backward_ex(None, _lib.ptr(c), _lib.ptr(o), b, h, w, levels, radius, None,
                                                 _lib.ptr_array(gp), 7, st) == -1
    torch.cuda.synchronize()


def ctypes_stream():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def test_lookup_autograd_refuses_coordinates_that_require_grad(T):
    from tf_raft_b200.train import _GridLookup
    coords = torch.zeros((1, 8, 8, 2), device='cuda', requires_grad=True)
    pyr = [torch.zeros((64, 8 >> l, 8 >> l), device='cuda') for l in range(4)]
    with pytest.raises(ValueError, match='detach'):
        _GridLookup.apply(coords, 4, *pyr)
    _GridLookup.apply(coords.detach(), 4, *pyr)


# --------------------------------------------------------------------------------------------- 2. optimiser rules
@pytest.mark.parametrize('clip', [0.0, 0.5, 1e6])
def test_torch_adamw_rule_vs_fp64_torch(T, clip):
    from tf_raft_b200 import _lib
    rng = np.random.default_rng(3)
    n = 100003
    p0 = rng.standard_normal(n).astype(F32)
    ref = torch.from_numpy(p0).double().requires_grad_(True)
    lr_sched = T.OneCycleLR(1e-3, 100)                     # warm-up over steps 0..4, then down
    opt = torch.optim.AdamW([ref], lr=1e-3, weight_decay=1e-4, eps=1e-8, foreach=False)
    sched = torch.optim.lr_scheduler.OneCycleLR(opt, 1e-3, 100, pct_start=0.05, cycle_momentum=False,
                                                anneal_strategy='linear')
    p, m, v = dev(p0), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
    sumsq, part = torch.zeros(1, device='cuda'), torch.zeros(1024, device='cuda')
    for t in range(1, 7):
        g = (rng.standard_normal(n) * (1e-3 if t % 2 else 1e-2)).astype(F32)
        gd = dev(g)
        _lib.call('sumsq', 'cuda', _lib.ptr(gd), n, _lib.ptr(part), 1024, _lib.ptr(sumsq))
        lr = lr_sched(t - 1)
        assert lr == opt.param_groups[0]['lr']
        _lib.call('adamw_step_ex', 'cuda', _lib.ptr(p), _lib.ptr(gd), _lib.ptr(m), _lib.ptr(v), n, _lib.ptr(sumsq), clip,
                  lr, 0.9, 0.999, 1e-8, 1e-4, 1 - 0.9 ** t, 1 - 0.999 ** t, 1)
        ref.grad = torch.from_numpy(g).double()
        if clip > 0:
            torch.nn.utils.clip_grad_norm_([ref], clip)
        opt.step()
        sched.step()
        st = opt.state[ref]
        # fp32 arithmetic: 1 - beta_2 = 0.001 is 4.7e-5 off in fp32, which moves v by as much relative, the Adam term
        # by half that; p's own rounding is an ulp of the largest entry
        for name, got, want, tol in (('p', p, ref.detach(), 1e-4 * lr + 4e-7 * float(ref.detach().abs().max())),
                                     ('m', m, st['exp_avg'], 1e-5 * float(st['exp_avg'].abs().max())),
                                     ('v', v, st['exp_avg_sq'], 1e-4 * float(st['exp_avg_sq'].abs().max()))):
            err = float((got.cpu().double() - want).abs().max())
            assert err <= tol, f'step {t} {name}: error {err:.3e}, tolerance {tol:.3e}'


def test_tfa_rule_through_ex_equals_adamw_step(T):
    from tf_raft_b200 import _lib
    rng = np.random.default_rng(5)
    n = 65537
    init = [rng.standard_normal(n).astype(F32) for _ in range(3)]
    init[2] = np.abs(init[2])
    g = dev(rng.standard_normal(n).astype(F32))
    sumsq, part = torch.zeros(1, device='cuda'), torch.zeros(1024, device='cuda')
    _lib.call('sumsq', 'cuda', _lib.ptr(g), n, _lib.ptr(part), 1024, _lib.ptr(sumsq))
    res = []
    for fn in ('adamw_step', 'adamw_step_ex'):
        p, m, v = (dev(x) for x in init)
        args = [_lib.ptr(p), _lib.ptr(g), _lib.ptr(m), _lib.ptr(v), n, _lib.ptr(sumsq), 1.0, 3e-4, 0.9, 0.999, 1e-7, 1e-5]
        _lib.call(fn, 'cuda', *(args + ([0.1, 0.001, 0] if fn.endswith('_ex') else [])))
        res.append([x.cpu().numpy() for x in (p, m, v)])
    assert all(same_bits(a, b) for a, b in zip(*res))


# --------------------------------------------------------------------------------------------- 3. the training step
def _model(T, ckpt, tmp_path, train_precision='fp32', frozen=False, lr=2e-4, total=200, clip=1.0, iters=2):
    path = tmp_path / 'raft-synthetic.pth'
    torch.save(ckpt, path)
    m = T.RAFT(conventions='pytorch', precision='f16x2', device='cuda', iters=iters, iters_pred=iters)
    m.load_pytorch_weights(str(path))
    if frozen:
        m.freeze_bn()
    m.compile(optimizer=T.TorchAdamW(weight_decay=1e-4, learning_rate=T.OneCycleLR(lr, total)), clip_norm=clip,
              train_precision=train_precision)
    return m


def _batch(step, b=2, H=64, W=96):
    im1, im2 = cases.images(b, H, W, 3 + 2 * step, 4 + 2 * step)
    rng = np.random.default_rng(9 + step)
    flow = (rng.standard_normal((b, H, W, 2)) * 5).astype(F32)
    valid = rng.uniform(size=(b, H, W)) > 0.1
    return im1, im2, flow, valid


def _pt(T, model):
    """The model's parameters in PyTorch layout (no `module.` prefix), NumPy."""
    sd = T.to_pytorch_state_dict({k: v.detach().cpu().numpy() for k, v in model.state_dict().items()})
    return {k[len('module.'):]: v.numpy() for k, v in sd.items()}


def _to_project(T, grads):
    """{PyTorch name: tensor} of trainable entries -> {project name: ndarray} (fnet norms excluded)."""
    sd = {k: v.detach().float().numpy() for k, v in grads.items()}
    for k in list(sd):
        if '.downsample.1.' in k:
            sd[k.replace('.downsample.1.', '.norm3.')] = sd[k]
    out = T.load_pytorch_checkpoint(sd)
    return {k: v for k, v in out.items() if not (k.startswith('fnet.') and k.endswith(('.gamma', '.beta')))}


@pytest.mark.parametrize('train_precision', ['fp32', 'f16x2'])
@pytest.mark.parametrize('bn', ['train', 'frozen'])
def test_three_train_steps_vs_torch(T, ckpt, tmp_path, bn, train_precision):
    """Three train_steps at 64x96, batch 2, iters 2 against RAFT's training forward in float64 with the real torch
    AdamW, clip_grad_norm_ and OneCycleLR: per step the loss, the global norm, every gradient (per tensor and as a
    whole), the update where the gradient is well determined, Adam's m and v, and cnet's running statistics.  Each
    oracle gradient is taken at the model's parameters before the step (see test_gpu_train_state.py)."""
    lr, clip, iters = 2e-4, 1.0, 2
    model = _model(T, ckpt, tmp_path, train_precision, bn == 'frozen', lr=lr, clip=clip, iters=iters)
    oracle = pto.TorchStep(rp._sd(ckpt, torch.float64), lr, 1e-4, 200, clip)
    fnet0 = {k: v.clone() for k, v in model.state_dict().items() if k.startswith('fnet.') and k.endswith(('gamma', 'beta'))}
    run0 = {k: v.clone() for k, v in model.state_dict().items() if k.endswith(('moving_mean', 'moving_variance'))}
    for step in range(3):
        im1, im2, flow, valid = _batch(step)
        cur = _pt(T, model)
        oracle.load(cur)
        lr_t = oracle.opt.param_groups[0]['lr']
        loss_o, grads_o, norm_o = oracle.step(im1, im2, flow, valid, iters, bn)
        model.reset_metrics()
        out = model.train_step((dev(im1), dev(im2), dev(flow), torch.from_numpy(valid).cuda()))
        tr = model._trainer
        assert model.optimizer.iterations == step + 1
        assert out['loss'] == pytest.approx(loss_o, rel=2e-4), (step, out['loss'], loss_o)
        gnorm = math.sqrt(float((tr.flat.g.double() ** 2).sum()))
        assert gnorm == pytest.approx(norm_o, rel=1e-3), (step, gnorm, norm_o)
        want_g = _to_project(T, grads_o)
        assert sorted(want_g) == sorted(tr.flat.views), 'trainable sets differ'
        num = den = 0.0
        for k, want in want_g.items():
            got = tr.flat.views[k].grad.cpu().numpy()
            num += float(((got - want).astype(np.float64) ** 2).sum())
            den += float((want.astype(np.float64) ** 2).sum())
            tol = 5e-2 * float(np.abs(want).max()) + 2e-6
            assert float(np.abs(got - want).max()) <= tol, f'step {step + 1} gradient of {k}'
        assert math.sqrt(num / den) <= 1e-2, f'step {step + 1}: relative L2 error of the gradient'
        new_o = _to_project(T, {k: oracle.sd[k] for k in oracle.names})
        old = _to_project(T, {k: torch.from_numpy(cur[k]) for k in oracle.names})
        new = {k: v.detach().cpu().numpy() for k, v in tr.flat.views.items()}
        for k, w in new_o.items():
            g = np.abs(want_g[k])
            sel = g >= 0.2 * g.max()
            if float(g.max()) < 1e-5:
                continue
            err = float(np.abs((new[k] - old[k]) - (w - old[k]))[sel].max()) / lr_t
            assert err <= 5e-2, f'step {step + 1} {k}: update differs by {err:.3f} x lr'
        # m is a sum of gradients, v of their squares: each within the gradient's tolerance of the tensor's scale
        # (biases in front of a norm layer have a zero true gradient: noise, as above)
        for slot, buf, rel in (('exp_avg', tr.flat.m, 0.1), ('exp_avg_sq', tr.flat.v, 0.2)):
            want_s = _to_project(T, oracle.slot(slot))
            got_s = tr.flat.slot(buf.cpu())
            for k, w in want_s.items():
                if float(np.abs(want_g[k]).max()) < 1e-5:
                    continue
                err = float(np.abs(got_s[k].numpy() - w).max())
                assert err <= rel * float(np.abs(w).max()) + 1e-12, f'step {step + 1} {slot} of {k}'
        for k, w in _to_project(T, {k: v for k, v in oracle.sd.items() if 'running' in k}).items():
            if k.endswith(('moving_mean', 'moving_variance')):
                got = tr.moving[k].cpu().numpy()
                assert float(np.abs(got - w).max()) <= 2e-5 * float(np.abs(w).max()), f'step {step + 1} {k}'
        print(f'{bn} {train_precision} step {step + 1}: loss {out["loss"]:.6f} (oracle {loss_o:.6f}), '
              f'norm {gnorm:.4f} (oracle {norm_o:.4f})')
    sd = model.state_dict()
    for k, v in fnet0.items():
        assert torch.equal(sd[k], v), f'{k} moved'
    if bn == 'frozen':
        for k, v in run0.items():
            assert torch.equal(sd[k], v), f'{k} changed under freeze_bn'
        assert model._num_batches_tracked == 0
    else:
        assert model._num_batches_tracked == 3


def _state(model):
    t = model._trainer
    return {k: v.detach().cpu().clone() for k, v in dict(p=t.flat.p, g=t.flat.g, m=t.flat.m, v=t.flat.v,
                                                          **t.moving).items()}


@pytest.mark.parametrize('train_precision', ['fp32', 'f16x2'])
@pytest.mark.parametrize('bn', ['train', 'frozen'])
def test_train_step_is_deterministic(T, ckpt, tmp_path, bn, train_precision):
    states = []
    for run in range(2):
        model = _model(T, ckpt, tmp_path, train_precision, bn == 'frozen')
        for step in range(2):
            im1, im2, flow, valid = _batch(step)
            if run == 1 and step == 1:
                torch.use_deterministic_algorithms(True)
            try:
                model.train_step((dev(im1), dev(im2), dev(flow), torch.from_numpy(valid).cuda()))
            finally:
                torch.use_deterministic_algorithms(False)
        states.append(_state(model))
    for k in states[0]:
        assert torch.equal(states[0][k], states[1][k]), k


def test_guards(T, ckpt, tmp_path):
    m = T.RAFT(conventions='pytorch', device='cuda')
    for opt in (None, T.AdamW(weight_decay=1e-4)):
        with pytest.raises(NotImplementedError, match='TorchAdamW'):
            m.compile(optimizer=opt)
    with pytest.raises(NotImplementedError, match='TorchAdamW'):
        m.train_step(None)
    with pytest.raises(NotImplementedError, match='UnsupervisedLoss'):
        m.compile(optimizer=T.TorchAdamW(1e-4, 1e-4), loss=T.UnsupervisedLoss())
    tf = T.RAFT(device='cuda')
    with pytest.raises(ValueError):
        tf.freeze_bn()
    with pytest.raises(ValueError):
        tf.save_pytorch_weights(str(tmp_path / 'x.pth'))
    tf.compile(optimizer=T.TorchAdamW(1e-4, 1e-4), clip_norm=1.0)
    with pytest.raises(TypeError):
        tf.train_step(tuple(dev(x) if x.dtype != bool else torch.from_numpy(x).cuda() for x in _batch(0, 1)))


# --------------------------------------------------------------------------------------------- 4. .pth export
def test_save_pytorch_weights_round_trip(T, ckpt, tmp_path):
    m = _model(T, ckpt, tmp_path)
    out = tmp_path / 'out.pth'
    m.save_pytorch_weights(str(out))
    got = torch.load(out, map_location='cpu', weights_only=True)
    assert sorted(got) == sorted(ckpt)
    for k, v in ckpt.items():
        if k.endswith('num_batches_tracked'):
            assert got[k].dtype == torch.int64 and got[k].shape == ()
            continue
        assert got[k].dtype == v.dtype and torch.equal(got[k], v), k


def test_trained_pth_reaches_the_original_inference(T, ckpt, tmp_path):
    """Three steps, save_pytorch_weights, and the file through RAFT's inference restated in float64: within the
    end-to-end gate (1e-3) of the trained model's own inference."""
    model = _model(T, ckpt, tmp_path, iters=3, lr=1e-3)
    for step in range(3):
        im1, im2, flow, valid = _batch(step)
        model.train_step((dev(im1), dev(im2), dev(flow), torch.from_numpy(valid).cuda()))
    out = tmp_path / 'trained.pth'
    model.save_pytorch_weights(str(out))
    trained = torch.load(out, map_location='cpu', weights_only=True)
    assert not torch.equal(trained['module.update_block.mask.2.weight'], ckpt['module.update_block.mask.2.weight'])
    assert int(trained['module.cnet.norm1.num_batches_tracked']) == 3
    im1, im2 = cases.images(2, 64, 96, 40, 41)
    want, _ = rp.forward(trained, im1, im2, iters=3)
    got = model([dev(im1), dev(im2)], training=False)
    err = max(float(np.abs(g.cpu().numpy() - w).max()) for g, w in zip(got, want))
    print(f'trained .pth vs fp64 RAFT inference: max abs {err:.2e}')
    assert err <= 1e-3


# --------------------------------------------------------------------------------------------- 5. fit, resume, script
@pytest.fixture(scope='module')
def chairs(tmp_path_factory):
    import test_gpu_fit as gf
    return gf._write_chairs(str(tmp_path_factory.mktemp('chairs')))


def test_resumed_fit_equals_uninterrupted(T, ckpt, tmp_path, chairs):
    import test_gpu_fit as gf
    full = _model(T, ckpt, tmp_path)
    full.freeze_bn()
    train, _ = gf._datasets(chairs, 5)
    full.fit(train.batches(gf.BATCH, workers=2, repeat=True), epochs=2, steps_per_epoch=gf.STEPS, verbose=0)
    first = _model(T, ckpt, tmp_path)
    first.freeze_bn()
    train, _ = gf._datasets(chairs, 5)
    stream = train.batches(gf.BATCH, workers=2, repeat=True)
    first.fit(stream, epochs=1, steps_per_epoch=gf.STEPS, verbose=0)
    prefix = str(tmp_path / 'resume' / 'model')
    first.save_weights(prefix)
    second = _model(T, rp.synthetic_checkpoint(seed=12), tmp_path)
    second.freeze_bn()
    second.load_weights(prefix)
    second.fit(stream, epochs=1, steps_per_epoch=gf.STEPS, verbose=0)
    assert second.optimizer.iterations == full.optimizer.iterations == 2 * gf.STEPS
    a, b = _state(full), _state(second)
    for k in a:
        if k != 'g':
            assert torch.equal(a[k], b[k]), k


def test_train_script_fine_tunes_a_pth(T, ckpt, tmp_path, chairs):
    yaml = pytest.importorskip('yaml', reason='scripts/train.py reads YAML configs and needs PyYAML')
    import test_gpu_fit as gf
    data, split = chairs
    src = tmp_path / 'raft-synthetic.pth'
    torch.save(ckpt, src)
    config = {'data': {'root': data, 'split_txt': split}, 'augment': gf.AUG,
              'model': {'iters': 2, 'iters_pred': 2, 'resume': 0},
              'train': {'epochs': 1, 'batch_size': gf.BATCH, 'learning_rate': 1e-4, 'weight_decay': 1e-5,
                        'clip_norm': 1.0},
              'visualize': {'num_visualize': 1, 'choose_random': False}, 'logdir': str(tmp_path / 'logs')}
    cfg = str(tmp_path / 'run.yml')
    with open(cfg, 'w') as f:
        yaml.dump(config, f)
    base = [sys.executable, os.path.join(ROOT, 'scripts', 'train.py'), 'chairs', cfg, '--workers', '2']
    proc = subprocess.run(base + ['--pytorch-checkpoint', str(src), '--freeze-bn', '--gamma', '0.85', '--seed', '1'],
                          capture_output=True, text=True, timeout=1200)
    assert proc.returncode == 0, proc.stdout[-3000:] + proc.stderr[-3000:]
    (logdir,) = glob.glob(os.path.join(config['logdir'], '*'))
    path = os.path.join(logdir, 'checkpoints', 'model.pth')
    m = T.RAFT(conventions='pytorch', device='cuda')
    m.load_pytorch_weights(path)
    sd = torch.load(path, map_location='cpu', weights_only=True)
    assert sorted(sd) == sorted(ckpt)
    assert all(torch.equal(sd[k], ckpt[k]) for k in ckpt if 'running' in k), 'freeze_bn: running statistics moved'
    bad = subprocess.run(base + ['--pytorch-checkpoint', str(src), '--small'], capture_output=True, text=True)
    assert bad.returncode != 0 and '--small' in bad.stderr
