"""The NumPy float32 emulations of the training step's two fixed-order backward kernels (oracle/determinism_np.py) against
float64 autograd, and the upsampling emulation's NaN cells against PyTorch's own backward.  The GPU tests hold the
kernels to these emulations bit for bit (tests/test_gpu_determinism.py)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cases
from oracle import determinism_np as dn, raft_torch as rt

F64 = torch.float64
# the (radius, levels) pairs of the lookup's fp64 test in tests/test_gpu_geometry.py
LOOKUP_CONFIGS = ((3, 4), (4, 4), (2, 1), (4, 5), (0, 2), (5, 6))
KINDS = ('grid', 'jitter', 'edge')
UP_SHAPES = ((2, 5, 7), (1, 1, 6), (2, 4, 1), (1, 1, 1), (3, 9, 13))


def lookup_pyramid(b, h, w, levels, seed=30):
    """fp32 pyramid of the oracle CorrBlock, as NumPy (M, h_l, w_l, 1) levels."""
    f1, f2 = cases.fmaps(b, h, w, 64, seed=seed + h + w)
    return [np.ascontiguousarray(p.numpy()) for p in rt.CorrBlock(torch.from_numpy(f1), torch.from_numpy(f2), levels, 0).corr_pyramid]


def oracle_lookup_grads(pyr, coords, g, radius, dtype=F64):
    P = [torch.from_numpy(p).to(dtype).requires_grad_(True) for p in pyr]
    c = torch.from_numpy(coords).to(dtype).requires_grad_(True)
    cb = rt.CorrBlock.__new__(rt.CorrBlock)
    cb.corr_pyramid, cb.num_levels, cb.radius = P, len(P), radius
    cb.retrieve(c).backward(torch.from_numpy(g).to(dtype))
    return c.grad.numpy(), [q.grad.numpy() for q in P]


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('radius,levels', LOOKUP_CONFIGS)
def test_lookup_emulation_vs_fp64_autograd(radius, levels, kind):
    """d/d coords and d/d pyramid of the fixed-order emulation against autograd of the oracle sampler in fp64, within
    the tolerances the GPU lookup backward is held to (tests/test_gpu_geometry.py)."""
    for b, h, w in cases.LOOKUP_GRIDS[levels]:
        pyr = lookup_pyramid(b, h, w, levels)
        coords = cases.lookup_coords(b, h, w, kind)
        g = np.random.default_rng(5).standard_normal((b, h, w, levels * (2 * radius + 1) ** 2)).astype(np.float32)
        gc64, gp64 = oracle_lookup_grads(pyr, coords, g, radius)
        gc, gp = dn.lookup_backward(pyr, coords, g, radius)
        np.testing.assert_allclose(gc, gc64.reshape(-1, 2), atol=2e-4, rtol=1e-4)
        for l in range(levels):
            np.testing.assert_allclose(gp[l], gp64[l][..., 0], atol=1e-5, rtol=1e-5, err_msg=f'level {l}')


def test_lookup_emulation_accumulates_into_its_inputs():
    """Non-zero accumulators on entry: touched cells end as in + the terms, untouched cells and coordinates keep their
    bits exactly."""
    b, h, w, levels, radius = 2, 9, 13, 4, 3
    pyr = lookup_pyramid(b, h, w, levels)
    coords = cases.lookup_coords(b, h, w, 'jitter')
    g = np.random.default_rng(6).standard_normal((b, h, w, levels * (2 * radius + 1) ** 2)).astype(np.float32)
    rng = np.random.default_rng(7)
    gc_in = rng.standard_normal((b * h * w, 2)).astype(np.float32)
    gp_in = [rng.standard_normal(p.shape[:3]).astype(np.float32) for p in pyr]
    gc0, gp0 = dn.lookup_backward(pyr, coords, g, radius)
    gc1, gp1 = dn.lookup_backward(pyr, coords, g, radius, gc_in, gp_in)
    np.testing.assert_allclose(gc1, gc_in + gc0, atol=1e-4, rtol=1e-5)
    for l in range(levels):
        untouched = gp0[l] == 0
        assert untouched.any() and (l == levels - 1 or (~untouched).any())      # the last level is 1 x 1: no weight
        assert np.array_equal(gp1[l][untouched], gp_in[l][untouched])
        np.testing.assert_allclose(gp1[l], gp_in[l] + gp0[l], atol=1e-5, rtol=1e-5)


def _torch_up(flow_nhwc, dtype):
    """The training graph's upsampling (before its factor 8) and its input, NCHW, in `dtype`."""
    x = torch.from_numpy(flow_nhwc).to(dtype).permute(0, 3, 1, 2).requires_grad_(True)
    return x, F.interpolate(x, scale_factor=8, mode='bilinear', align_corners=False)


@pytest.mark.parametrize('shape', UP_SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_upflow8_emulation_vs_fp64_autograd(shape):
    b, h, w = shape
    rng = np.random.default_rng(h * 31 + w)
    flow = rng.standard_normal((b, h, w, 2)).astype(np.float32)
    g = rng.standard_normal((b, 8 * h, 8 * w, 2)).astype(np.float32)
    x, up = _torch_up(flow, F64)
    up.backward(torch.from_numpy(g).to(F64).permute(0, 3, 1, 2))
    want = x.grad.permute(0, 2, 3, 1).numpy()
    got = dn.upflow8_backward(g)
    assert got.dtype == np.float32 and got.shape == (b, h, w, 2)
    np.testing.assert_allclose(got, want, atol=1e-5, rtol=1e-5)


@pytest.mark.parametrize('shape', UP_SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_upflow8_emulation_nan_cells_match_torch(shape):
    """NaN and +-inf planted in the output gradient, at image corners and edges (where a corner's weight is zero) and
    inside: the emulation's NaN cells are exactly those of PyTorch's CPU backward, and its other cells are finite where
    torch's are."""
    b, h, w = shape
    rng = np.random.default_rng(3)
    g = rng.standard_normal((b, 8 * h, 8 * w, 2)).astype(np.float32)
    H, W = 8 * h, 8 * w
    for Y, X, v in ((0, 0, np.nan), (H - 1, W - 1, np.inf), (3, W // 2, -np.inf), (H // 2, 2, np.nan),
                    (H - 2, 0, np.nan), (H // 3, W - 4, np.inf)):
        g[-1, Y, X, (Y + X) % 2] = v
    x, up = _torch_up(np.zeros((b, h, w, 2), np.float32), torch.float32)
    up.backward(torch.from_numpy(g).permute(0, 3, 1, 2))
    want = x.grad.permute(0, 2, 3, 1).numpy()
    got = dn.upflow8_backward(g)
    assert np.isnan(want).any()
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.array_equal(np.isfinite(got), np.isfinite(want))
