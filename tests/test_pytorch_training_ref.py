"""The test infrastructure of RAFT(conventions='pytorch') training, on the CPU: the NumPy float32 emulation of the
grid_sample lookup backward against float64 autograd of F.grid_sample, OneCycleLR against torch's scheduler, and the
restated training forward against the inference restatement."""
import numpy as np
import pytest
import torch

import cases
import pytorch_train_oracle as pto
from oracle import raft_pytorch as rp

F32 = np.float32


def _coords(b, h, w, kind):
    if kind in ('grid', 'jitter', 'edge'):
        return cases.lookup_coords(b, h, w, kind)
    c = cases.lookup_coords(b, h, w, 'jitter')             # 'far': every tap outside the level, or nearly so
    c[..., 0] += np.where(c[..., 0] > w / 2, F32(3 * w), F32(-3 * w))
    c[..., 1][::2] -= F32(1000)
    return c.astype(F32)


@pytest.mark.parametrize('levels,shape', [(lv, s) for lv, shapes in cases.LOOKUP_GRIDS.items() for s in shapes])
@pytest.mark.parametrize('radius', [4, 3, 2])
@pytest.mark.parametrize('kind', ['grid', 'jitter', 'edge', 'far'])
def test_lookup_backward_emulation_vs_fp64_autograd(levels, shape, radius, kind):
    """d loss / d pyramid of the grid_sample lookup: the float32 emulation is within a few ulps of sum |w * go| of
    float64 autograd through RAFT's bilinear_sampler (F.grid_sample, align_corners=True), plus the float32
    normalisation's rounding of the weights: ix = fl((2v / (n-1) - 1 + 1) / 2 * (n-1)) is within a few ulps of
    max(|v|, n) of v, which moves each weight by as much (so a corner that float64 reaches with weight 0 may receive a
    term of that size, and an integer v gives weights 1 - d, d)."""
    b, h, w = shape
    rng = np.random.default_rng(levels * 100 + radius * 10 + len(kind))
    coords = _coords(b, h, w, kind)
    pyr = [torch.zeros((b * h * w, 1, h >> l, w >> l), dtype=torch.float64, requires_grad=True) for l in range(levels)]
    go = rng.standard_normal((b, h, w, levels * (2 * radius + 1) ** 2)).astype(F32)
    c64 = torch.from_numpy(coords).double().permute(0, 3, 1, 2)
    out = rp.corr_lookup(pyr, c64, radius)
    want = torch.autograd.grad(out, pyr, torch.from_numpy(go).double().permute(0, 3, 1, 2))
    scale = torch.autograd.grad(rp.corr_lookup(pyr, c64, radius), pyr,
                                torch.from_numpy(np.abs(go)).double().permute(0, 3, 1, 2))
    got = pto.lookup_backward_emulated(coords, go, [np.zeros(p.shape[:1] + p.shape[2:], F32) for p in pyr], radius)
    eps = float(np.finfo(F32).eps)
    for l in range(levels):
        wl, sl = want[l][:, 0].numpy(), scale[l][:, 0].numpy()
        err = np.abs(got[l].astype(np.float64) - wl)
        a = np.abs(go.reshape(b * h * w, levels, -1)[:, l].astype(np.float64)).sum(-1)     # sum |go| of the taps
        c = np.abs(coords.reshape(-1, 2).astype(np.float64)) / 2 ** l + radius
        v = np.where(np.isfinite(c), c, 0).max(-1) + max(h >> l, w >> l)
        tol = 8 * eps * sl + 4 * eps * (v * a)[:, None, None] + 1e-30
        assert (err <= tol).all(), f'level {l}: max error / tolerance {float((err / tol).max()):.2f}'


def test_lookup_backward_emulation_leaves_untouched_cells():
    """A level of size 1 receives nothing, and the accumulators' other cells keep their values (NaN included)."""
    b, h, w = 1, 5, 7
    coords = cases.lookup_coords(b, h, w, 'jitter')
    init = [np.full((b * h * w, h >> l, w >> l), np.nan, F32) for l in range(3)]
    go = np.ones((b, h, w, 3 * 81), F32)
    got = pto.lookup_backward_emulated(coords, go, init, 4)
    assert got[2].shape[1] == 1 and np.isnan(got[2]).all()                      # 5 >> 2 = 1 row
    assert np.isnan(got[0]).all()                                              # NaN + anything stays NaN


def test_one_cycle_lr_equals_torch():
    from tf_raft_b200 import OneCycleLR
    for max_lr, total in ((4e-4, 220), (1.25e-4, 100100 // 50), (1e-3, 21)):
        opt = torch.optim.AdamW([torch.zeros(1, requires_grad=True)], lr=max_lr)
        sched = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr, total, pct_start=0.05, cycle_momentum=False,
                                                    anneal_strategy='linear')
        ours = OneCycleLR(max_lr, total)
        for k in range(total + 1):
            assert ours(k) == opt.param_groups[0]['lr'], (max_lr, total, k)
            if k < total:
                opt.step()
                sched.step()
        with pytest.raises(ValueError):
            sched.step()
        with pytest.raises(ValueError):
            ours(total + 1)


def test_train_forward_frozen_equals_inference_restatement():
    """With BatchNorm frozen and no gradient, the training restatement computes RAFT's inference exactly (fp64)."""
    sd = rp._sd(rp.synthetic_checkpoint(seed=3), torch.float64)
    im1, im2 = cases.images(1, 64, 96, 5, 6)
    want, _ = rp.forward(sd, im1, im2, iters=3)
    with torch.no_grad():
        got = pto.train_forward(dict(sd), im1, im2, 3, bn='frozen')
    assert len(got) == 3
    for g, w in zip(got, want):
        assert np.array_equal(g.numpy(), w)


def test_train_forward_updates_running_statistics_with_momentum_0_1():
    sd = rp._sd(rp.synthetic_checkpoint(seed=3), torch.float64)
    before = {k: v.clone() for k, v in sd.items() if 'running' in k}
    im1, im2 = cases.images(2, 64, 64, 5, 6)
    with torch.no_grad():
        pto.train_forward(sd, im1, im2, 1, bn='train')
    x = 2 * (torch.from_numpy(im1).double().permute(0, 3, 1, 2) / 255.0) - 1.0
    stem = rp._conv(sd, x, 'cnet.conv1', 2)
    mean, var = stem.mean(dim=(0, 2, 3)), stem.var(dim=(0, 2, 3), unbiased=True)
    torch.testing.assert_close(sd['cnet.norm1.running_mean'], 0.9 * before['cnet.norm1.running_mean'] + 0.1 * mean)
    torch.testing.assert_close(sd['cnet.norm1.running_var'], 0.9 * before['cnet.norm1.running_var'] + 0.1 * var)


def test_to_pytorch_state_dict_inverts_the_loader():
    """load_pytorch_checkpoint then to_pytorch_state_dict gives the checkpoint back key for key and bit for bit, apart
    from num_batches_tracked (the count given); fnet's fixed norm gamma / beta write no entries."""
    from tf_raft_b200 import load_pytorch_checkpoint, to_pytorch_state_dict
    ck = rp.synthetic_checkpoint(seed=3)
    params = load_pytorch_checkpoint(ck)
    assert 'fnet.norm1.gamma' in params
    out = to_pytorch_state_dict(params, 7)
    assert list(out) != [] and sorted(out) == sorted(ck)
    for k, v in ck.items():
        if k.endswith('num_batches_tracked'):
            assert out[k].dtype == torch.int64 and int(out[k]) == 7
        else:
            assert out[k].dtype == v.dtype and torch.equal(out[k], v), k
    with pytest.raises(ValueError):
        to_pytorch_state_dict({'fnet.conv1.weird': np.zeros(3, F32)})
