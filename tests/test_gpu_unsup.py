"""Self-supervised training on the GPU: the census kernel bit for bit against NumPy float32, the fused loss-and-gradient
kernel against the float64 restatement (oracle/unsup_np.py), one unsupervised train_step against the same step done with
torch.autograd on the oracle forward, `fit` with UnsupervisedLoss, and a loss that goes down on translated pairs."""
import math

import numpy as np
import pytest
import torch

import cases
from oracle import raft_torch as rt, train_ref, unsup_np, weights

pytestmark = pytest.mark.gpu
F32 = np.float32
FROZEN = ('moving_mean', 'moving_variance')


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _texture(b, h, w, seed, smooth=True):
    """Random RGB in 0..255; smooth=True blurs it so that a census window sees structure, not only noise."""
    im = np.random.default_rng(seed).uniform(0, 255, (b, h, w, 3))
    if smooth:
        from scipy.ndimage import uniform_filter
        im = uniform_filter(im, size=(1, 3, 3, 1), mode='wrap')
    return im.astype(F32)


# --------------------------------------------------------------------------------------------- census
@pytest.mark.parametrize('shape', [(2, 13, 17), (1, 5, 9), (3, 9, 4), (1, 6, 6), (1, 1080, 2560)],
                         ids=['odd', 'H<7', 'W<7', 'both<7', '1080x2560'])
def test_census_matches_numpy_bit_for_bit(shape):
    from tf_raft_b200.losses import census_transform
    im = _texture(*shape, seed=sum(shape), smooth=False)
    got = census_transform(dev(im)).cpu().numpy()
    np.testing.assert_array_equal(got, unsup_np.census(im))


def test_census_nan_pixel_reaches_exactly_the_windows_that_cover_it():
    from tf_raft_b200.losses import census_transform
    b, h, w, (ny, nx) = 2, 19, 23, (9, 4)
    im = _texture(b, h, w, 3, smooth=False)
    im[1, ny, nx, 2] = np.nan
    got = census_transform(dev(im)).cpu().numpy()
    np.testing.assert_array_equal(got, unsup_np.census(im))
    nan = np.isnan(got)
    assert not nan[0].any()
    want = np.zeros((h, w, 48), dtype=bool)
    want[ny, nx, :] = True                                          # its own vector: t = g(neighbour) - NaN
    for k, (dy, dx) in enumerate(unsup_np.OFFSETS):
        y, x = ny - dy, nx - dx                                     # the pixel whose k-th neighbour is the NaN pixel
        if 0 <= y < h and 0 <= x < w:
            want[y, x, k] = True
    np.testing.assert_array_equal(nan[1], want)


# --------------------------------------------------------------------------------------------- loss and gradient
def _flows(case, n, b, h, w, rng):
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing='ij')
    out = []
    for i in range(n):
        f = (rng.standard_normal((b, h, w, 2)) * 2.5).astype(F32)
        if case == 'integer':                                        # landings on texels, on W-1 and on H-1
            f = np.round(f)
            f[:, :, ::3, 0] = (w - 1 - xs)[:, ::3]
            f[:, ::4, :, 1] = (h - 1 - ys)[::4, :]
            f[:, 1::5, 1::5] = 0.0
        elif case == 'leaving' and i < n - 1:                         # intermediate predictions leave the frame
            f[:, ::2] *= 20
            f[:, 1::3, :, 0] = -(xs[1::3] + 0.5)
        elif case == 'flat':                                          # zero neighbour differences
            f[:, :, : w // 2] = f[:, :1, :1]
            f[:, h // 2:] = np.round(f[:, h // 2:])
            f[:, h // 2:, ::2] = f[:, h // 2:, 1::2][:, :, : (w + 1) // 2]
        elif case == 'nonfinite':
            f[0, 5, 7, 0] = np.nan
            f[1, 9, 11, 1] = np.inf if i % 2 else -np.inf
            f[1, 2, 3] = np.inf
        out.append(f)
    return out


def _gpu_loss(im1, im2, fw, bw, loss_fn):
    pf = [dev(f).requires_grad_(True) for f in fw]
    pb = [dev(f).requires_grad_(True) for f in bw]
    loss = loss_fn((dev(im1), dev(im2)), (pf, pb))
    grads = torch.autograd.grad(loss, pf + pb)
    return loss.detach(), [g.cpu().numpy() for g in grads]


@pytest.mark.parametrize('case', ['random', 'integer', 'leaving', 'flat', 'nonfinite'])
def test_loss_and_gradient_match_fp64_oracle(case):
    from tf_raft_b200 import UnsupervisedLoss
    b, h, w, n = 2, 24, 40, 3
    rng = np.random.default_rng(len(case))
    im1 = _texture(b, h, w, 1)
    im2 = _texture(b, h, w, 2)
    if case == 'flat':
        im1[:, :, : w // 3] = 128.0                                 # zero image differences: edge weight 1
    fw, bw = _flows(case, n, b, h, w, rng), _flows(case, n, b, h, w, rng)
    loss_fn = UnsupervisedLoss(census_weight=1.0, smoothness_weight=0.5)
    loss, grads = _gpu_loss(im1, im2, fw, bw, loss_fn)
    leaves = [torch.from_numpy(f).double().requires_grad_(True) for f in fw + bw]
    want = unsup_np.loss(im1, im2, leaves[:n], leaves[n:])
    want_g = torch.autograd.grad(want, leaves)
    got, want = float(loss), float(want.detach())
    if case == 'nonfinite':             # NaN / inf reach the loss; d|u|/du is 0 at NaN in autograd, so not the gradient
        assert math.isnan(got) and math.isnan(want)
    else:
        assert got == pytest.approx(want, rel=1e-5), (got, want)
    finite = [np.isfinite(g.numpy()) for g in want_g]
    scale = max(float(np.abs(g.numpy()[m]).max()) for g, m in zip(want_g, finite))
    worst = 0.0
    for i, (g, wg, m) in enumerate(zip(grads, want_g, finite)):
        wg = wg.numpy()
        np.testing.assert_array_equal(np.isnan(g), np.isnan(wg), err_msg=f'prediction {i}: NaN pattern')
        np.testing.assert_array_equal(np.isinf(g), np.isinf(wg), err_msg=f'prediction {i}: inf pattern')
        err = float(np.abs(g[m] - wg[m]).max())
        worst = max(worst, err)
        assert err <= 1e-5 * scale, f'prediction {i}: gradient error {err:.3e} (scale {scale:.3e})'
    print(f'{case}: loss {got:.8g} (oracle {want:.8g}), worst gradient error {worst / scale:.2e} of the largest')


def test_two_calls_are_bit_identical():
    from tf_raft_b200 import UnsupervisedLoss
    b, h, w, n = 2, 64, 96, 4
    rng = np.random.default_rng(0)
    im1, im2 = _texture(b, h, w, 5), _texture(b, h, w, 6)
    fw, bw = _flows('random', n, b, h, w, rng), _flows('random', n, b, h, w, rng)
    first = _gpu_loss(im1, im2, fw, bw, UnsupervisedLoss())
    second = _gpu_loss(im1, im2, fw, bw, UnsupervisedLoss())
    assert first[0].item() == second[0].item()
    for g1, g2 in zip(first[1], second[1]):
        assert g1.tobytes() == g2.tobytes()


def test_host_checks_reject_bad_arguments():
    from tf_raft_b200 import _lib
    x = torch.zeros((1, 8, 8, 48), device='cuda')
    im = torch.zeros((1, 8, 8, 3), device='cuda')
    occ = torch.zeros((1, 8, 8), dtype=torch.uint8, device='cuda')
    flows = torch.zeros((2, 1, 8, 8, 2), device='cuda')
    grad = torch.empty_like(flows)
    part = torch.zeros(64, dtype=torch.float64, device='cuda')
    sums = torch.zeros(4, dtype=torch.float64, device='cuda')

    def call(**kw):
        a = dict(ct=x, cs=x, n=2, h=8, w=8, cw=1.0, gamma=0.8, flows=flows)
        a.update(kw)
        _lib.call('unsup_loss', x.device, _lib.ptr(a['ct']), _lib.ptr(a['cs']), _lib.ptr(im), _lib.ptr(occ),
                  _lib.ptr(a['flows']), a['n'], 1, a['h'], a['w'], a['cw'], 0.5, 150.0, a['gamma'], _lib.ptr(part),
                  part.numel(), _lib.ptr(sums), _lib.ptr(grad))
    call()
    for kw, code in ((dict(ct=None), -1), (dict(cw=-1.0), -1), (dict(gamma=float('nan')), -1),
                     (dict(cs=x.view(-1)[1:]), -1), (dict(n=0), -2), (dict(h=1), -2)):
        with pytest.raises(RuntimeError, match=rf'\[{code}\]'):
            call(**kw)


# --------------------------------------------------------------------------------------------- the training step
def _oracle_unsup_step(params, im1, im2, variant, iters, clip_norm, lr, wd, beta1=0.9, beta2=0.999, eps=1e-7):
    leaves = {k: torch.tensor(v, dtype=torch.float32, requires_grad=not k.endswith(FROZEN)) for k, v in params.items()}
    rec = {}
    preds = rt.forward(leaves, np.concatenate([im1, im2]), np.concatenate([im2, im1]), variant, iters, training=True,
                       bn_record=rec)
    b = im1.shape[0]
    loss = unsup_np.loss(im1, im2, [p[:b] for p in preds], [p[b:] for p in preds])
    names = [k for k, v in leaves.items() if v.requires_grad]
    grads = [g.double() for g in torch.autograd.grad(loss, [leaves[k] for k in names])]
    norm = math.sqrt(sum(float((g ** 2).sum()) for g in grads))
    scale = clip_norm / max(norm, clip_norm)
    lr_t = lr * math.sqrt(1 - beta2) / (1 - beta1)
    new = {}
    for k, g in zip(names, grads):
        g = g * scale
        w = leaves[k].detach().double()
        w = w - wd * w
        new[k] = w - lr_t * ((1 - beta1) * g) / (((1 - beta2) * g * g).sqrt() + eps)
    return float(loss), norm, new, dict(zip(names, grads)), rec


@pytest.mark.parametrize('variant,shape,iters', [('small', (64, 96), 3), ('raft', (64, 96), 2)])
def test_unsupervised_train_step_vs_oracle_autograd(variant, shape, iters):
    """One RAFT.train_step with UnsupervisedLoss on (image1, image2) = the oracle step: loss (rel 2e-4), global norm
    (rel 1e-3), the update of every trainable variable where its gradient is well determined (5 % of lr, as
    tests/test_train.py), and (RAFT) cnet's moving statistics over the 2B images (2e-6 relative)."""
    import tf_raft_b200 as T
    from tf_raft_b200.train import AdamW
    H, W = shape
    bsz = 2
    p = weights.init_params(variant, 21, bias_scale=0.05, norm_jitter=0.1)
    im1, im2 = cases.images(bsz, H, W, 3, 4)
    clip_norm, lr, wd = 1.0, 1e-4, 1e-5
    loss_o, norm_o, new_o, grads_o, rec = _oracle_unsup_step(p, im1, im2, variant, iters, clip_norm, lr, wd)
    model = (T.RAFT if variant == 'raft' else T.SmallRAFT)(iters=iters, iters_pred=iters, precision='f16x2')
    model.load_params(p)
    model.compile(optimizer=AdamW(weight_decay=wd, learning_rate=lr), clip_norm=clip_norm, loss=T.UnsupervisedLoss())
    out = model.train_step((dev(im1), dev(im2)))
    assert out['loss'] == pytest.approx(loss_o, rel=2e-4), (out['loss'], loss_o)
    assert out['epe'] == 0.0 and model.flow_metrics['epe'][1] == 0            # no ground truth: no metrics
    tr = model._trainer
    gnorm = math.sqrt(float((tr.flat.g.double() ** 2).sum()))
    assert gnorm == pytest.approx(norm_o, rel=1e-3), (gnorm, norm_o)
    got = {k: v.cpu().double() for k, v in model.state_dict().items()}
    worst = 0.0
    for k, want in new_o.items():
        g = grads_o[k]
        sel = g.abs() >= 0.2 * g.abs().max()
        if float(g.abs().max()) < 1e-5 or not bool(sel.any()):
            continue
        old = torch.from_numpy(np.asarray(p[k], dtype=F32)).double()
        err = float(((got[k] - old) - (want - old))[sel].abs().max()) / lr
        worst = max(worst, err)
        assert err <= 5e-2, f'{k}: update differs by {err:.3f} x lr'
    worst_mov = 0.0
    if variant == 'raft':
        moving_ref = train_ref.bn_moving_update({k: np.asarray(v, dtype=np.float64) for k, v in p.items()
                                                 if k.endswith(FROZEN)}, rec)
        assert moving_ref
        for k, w in moving_ref.items():
            err = float(np.abs(tr.moving[k].double().cpu().numpy() - w).max()) / float(np.abs(w).max())
            worst_mov = max(worst_mov, err)
            assert err <= 2e-6, f'{k}: relative error {err:.2e}'
        assert rec['cnet.norm1'][2] == 2 * bsz * (H // 2) * (W // 2)          # BatchNorm over the 2B images
    print(f'{variant}: loss {out["loss"]:.6f} (oracle {loss_o:.6f}), norm {gnorm:.4f} (oracle {norm_o:.4f}), worst '
          f'update error {worst:.3f} x lr, worst moving-statistics error {worst_mov:.2e}')


def test_unsupervised_step_with_ground_truth_reports_forward_metrics():
    """(image1, image2, flow, valid): epe / u1 / u3 / u5 of the forward final prediction are updated."""
    import tf_raft_b200 as T
    from tf_raft_b200.train import AdamW
    im1, im2 = cases.images(2, 64, 96, 3, 4)
    flow = np.zeros((2, 64, 96, 2), dtype=F32)
    model = T.SmallRAFT(iters=2, iters_pred=2, seed=0)
    model.compile(optimizer=AdamW(weight_decay=1e-5, learning_rate=1e-4), clip_norm=1.0, loss=T.UnsupervisedLoss())
    out = model.train_step((dev(im1), dev(im2), dev(flow), torch.ones((2, 64, 96), device='cuda')))
    assert model.flow_metrics['epe'][1] == 1 and math.isfinite(out['epe']) and out['epe'] > 0
    assert math.isfinite(out['loss'])


# --------------------------------------------------------------------------------------------- fit and a falling loss
def _shifted_pairs(n, b, h, w, shift, seed):
    """Pairs whose second image is the first moved by `shift` = (dx, dy) px (wrapping), with that flow as ground truth."""
    out = []
    for i in range(n):
        im1 = _texture(b, h, w, seed + i)
        im2 = np.roll(im1, shift=(shift[1], shift[0]), axis=(1, 2))
        flow = np.broadcast_to(np.array(shift, dtype=F32), (b, h, w, 2)).copy()
        out.append((dev(im1), dev(im2), dev(flow), torch.ones((b, h, w), device='cuda')))
    return out


def test_fit_with_unsupervised_loss_logs_finite_loss_and_val_epe():
    import tf_raft_b200 as T
    from tf_raft_b200.train import AdamW
    train = _shifted_pairs(3, 2, 64, 96, (3, 1), 10)
    val = _shifted_pairs(2, 1, 64, 96, (2, -1), 20)
    model = T.SmallRAFT(iters=3, iters_pred=3, seed=1)
    model.compile(optimizer=AdamW(weight_decay=1e-5, learning_rate=1e-4), clip_norm=1.0, loss=T.UnsupervisedLoss())
    hist = model.fit([(a, b) for a, b, _, _ in train], epochs=2, validation_data=val, verbose=0)
    assert len(hist.history['loss']) == 2 and model.optimizer.iterations == 6
    for e in range(2):
        assert math.isfinite(hist.history['loss'][e]) and math.isfinite(hist.history['val_epe'][e])
    print('history', {k: [round(v, 4) for v in vs] for k, vs in hist.history.items()})


def test_loss_falls_on_translated_pairs():
    """30 steps over four pairs related by a translation of (2, 1) px: the mean loss of the last 5 steps is below that
    of the first 5.  A sanity check of the training loop, not of what is learned: the loss has no occlusion penalty, and
    from this random start the predictions may also lower it by making pixels occluded (DESIGN.md section 9.1)."""
    import tf_raft_b200 as T
    from tf_raft_b200.train import AdamW
    pairs = _shifted_pairs(4, 2, 64, 96, (2, 1), 30)
    model = T.SmallRAFT(iters=4, iters_pred=4, seed=2)
    model.compile(optimizer=AdamW(weight_decay=1e-5, learning_rate=2e-4), clip_norm=1.0, loss=T.UnsupervisedLoss())
    losses = []
    for s in range(30):
        a, b, _, _ = pairs[s % 4]
        model.reset_metrics()
        losses.append(model.train_step((a, b))['loss'])
    first, last = float(np.mean(losses[:5])), float(np.mean(losses[-5:]))
    print(f'mean loss, first 5 steps {first:.5f}, last 5 {last:.5f}')
    assert all(math.isfinite(v) for v in losses) and last < first
