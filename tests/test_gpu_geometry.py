"""Every geometry the host code can pick, against the oracle run in float64.

The host code picks a code path from the shape it is given: the pixel tile of every tensor-core convolution
(tc_pick_tile, and with it the halo of each mega-kernel dependency), the pyramid preparation (one fused kernel up to 4
levels, per-level pooling beyond), the lookup kernel (the window kernel at (radius, levels) = (4, 4) and (3, 4), with or
without 128-bit loads, the generic kernel elsewhere), and odd intermediate sizes in the stride-2 encoders.  The tests
below run each public layer at shapes that reach every one of those paths (tests/cases.py lists them) and compare it with
`oracle.raft_torch` in torch.float64, with the tolerances the model-shape tests use.  Each comparison also prints the fp32
oracle's error against the same fp64 truth, which shows how much of the tolerance an fp32 computation needs by itself.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import cases
from oracle import corr_np, raft_torch as rt, weights

pytestmark = pytest.mark.gpu
PRECISIONS = ('f16x2', 'fp32')
F64 = torch.float64
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))


def dev(a):
    if isinstance(a, torch.Tensor):
        return a.detach().float().contiguous().cuda()
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def maxabs(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max())


def nchw(a, dtype):
    return torch.from_numpy(a).permute(0, 3, 1, 2).to(dtype)


def nhwc(t):
    return None if t is None else t.permute(0, 2, 3, 1)


@pytest.fixture(scope='module')
def T():
    import tf_raft_b200
    from tf_raft_b200 import _lib
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    return tf_raft_b200


def _grid_id(g):
    return 'x'.join(map(str, g))


# --------------------------------------------------------------------------------------------- 1. update blocks per tile
UPDATE_TOL = dict(net=5e-5, mask=2e-4, delta=2e-4)      # the teacher-forced tolerances of tests/test_gpu_stages.py


@pytest.fixture(scope='module')
def update_truth():
    """(variant, grid) -> (params, inputs, fp64 outputs, fp32 outputs) of the oracle update block, computed once."""
    cache = {}

    def get(variant, grid):
        if (variant, grid) not in cache:
            b, h, w = grid
            p = weights.init_params(variant, 1234, bias_scale=0.05)
            ins = cases.update_inputs(variant, b, h, w, seed=20 + h * w)
            fn = rt.basic_update_block if variant == 'raft' else rt.small_update_block
            outs = []
            for dtype in (F64, torch.float32):
                net, mask, delta = fn(rt.Ops(p, dtype), *[nchw(a, dtype) for a in ins])
                outs.append(dict(net=nhwc(net), mask=nhwc(mask), delta=nhwc(delta)))
            cache[(variant, grid)] = (p, ins, outs[0], outs[1])
        return cache[(variant, grid)]
    return get


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('form', ['basic', 'basic-no-mask', 'small'])
@pytest.mark.parametrize('grid', cases.TILE_GRIDS, ids=_grid_id)
def test_update_block_every_tile_shape(T, update_truth, grid, form, precision):
    """One teacher-forced application of the update block per tensor-core tile shape (cases.TILE_GRIDS)."""
    variant = 'small' if form == 'small' else 'raft'
    p, ins, truth, fp32 = update_truth(variant, grid)
    blk = (T.BasicUpdateBlock if variant == 'raft' else T.SmallUpdateBlock)(precision=precision)
    blk.load_params(p, 'update_block.')
    args = [dev(a) for a in ins]
    net, mask, delta = blk(args, compute_mask=form == 'basic') if variant == 'raft' else blk(args)
    assert (mask is not None) == (form == 'basic')
    got = dict(net=net, mask=mask, delta=delta)
    errs = {k: (maxabs(got[k], truth[k]), maxabs(fp32[k], truth[k])) for k in got if got[k] is not None}
    tw, th = cases.tc_tile(grid[1], grid[2])
    print(f'{form} {precision} {_grid_id(grid)} (tile {tw}x{th}): ' +
          ', '.join(f'{k} {e:.2e} (fp32 oracle {o:.2e})' for k, (e, o) in errs.items()))
    for k, (e, _) in errs.items():
        assert e < UPDATE_TOL[k], (k, errs)


# --------------------------------------------------------------------------------------------- 2. correlation pyramid
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('case', cases.PYRAMID_CASES, ids=_grid_id)
def test_corr_pyramid_vs_fp64(T, case, precision):
    """CorrBlock's pyramid against the fp64 volume pooled the reference's way (corr.py:106-114)."""
    b, h, w, c, levels = case
    f1, f2 = cases.fmaps(b, h, w, c, seed=10 + c + levels)
    cb = T.CorrBlock(dev(f1), dev(f2), num_levels=levels, radius=4, precision=precision)
    truth = rt.CorrBlock(torch.from_numpy(f1).double(), torch.from_numpy(f2).double(), levels, 4).corr_pyramid
    fp32 = rt.CorrBlock(torch.from_numpy(f1), torch.from_numpy(f2), levels, 4).corr_pyramid
    assert len(cb.corr_pyramid) == levels
    for l, (lh, lw) in enumerate(cases.level_sizes(h, w, levels)):
        got = cb.corr_pyramid[l]
        assert tuple(got.shape) == (b * h * w, lh, lw, 1)
        print(f'{precision} {_grid_id(case)} level {l} ({lh}x{lw}): max-abs {maxabs(got, truth[l]):.2e} '
              f'(fp32 oracle {maxabs(fp32[l], truth[l]):.2e}), |corr| up to {float(truth[l].abs().max()):.2f}')
        np.testing.assert_allclose(got.cpu().numpy(), truth[l].numpy(), atol=2e-5, rtol=2e-5, err_msg=f'level {l}')


def test_tensor_core_pyramid_rejects_channels_not_a_multiple_of_64(T):
    """The tensor-core build reads C in 64-channel chunks: any other C is refused with an error, never a wrong pyramid.
    The fp32 build takes any C."""
    b, h, w, c, levels = 2, 9, 11, 96, 4
    f1, f2 = cases.fmaps(b, h, w, c)
    with pytest.raises(RuntimeError, match='bad shape'):
        T.CorrBlock(dev(f1), dev(f2), num_levels=levels, radius=4, precision='f16x2')
    cb = T.CorrBlock(dev(f1), dev(f2), num_levels=levels, radius=4, precision='fp32')
    truth = rt.CorrBlock(torch.from_numpy(f1).double(), torch.from_numpy(f2).double(), levels, 4).corr_pyramid
    for l in range(levels):
        np.testing.assert_allclose(cb.corr_pyramid[l].cpu().numpy(), truth[l].numpy(), atol=2e-5, rtol=2e-5)


# --------------------------------------------------------------------------------------------- 3. lookup
RADII = tuple(range(6))
KINDS = ('grid', 'jitter', 'edge')


def _oracle_pyramid(b, h, w, levels):
    """fp32 oracle pyramid as NumPy (M, h_l, w_l, 1) levels: the input both lookups are given."""
    f1, f2 = cases.fmaps(b, h, w, 64, seed=30 + h + w)
    pyr = rt.CorrBlock(torch.from_numpy(f1), torch.from_numpy(f2), levels, 0).corr_pyramid
    return [np.ascontiguousarray(p.numpy()) for p in pyr]


def _retrieve(T, pyr_dev, coords, radius):
    b, h, w, _ = coords.shape
    cb = T.CorrBlock.__new__(T.CorrBlock)
    cb.corr_pyramid, cb.num_levels, cb.radius, cb._shape = pyr_dev, len(pyr_dev), radius, (b, h, w)
    return cb.retrieve(dev(coords))


def lookup_forward_matrix(T, plant=None):
    """CorrBlock.retrieve bit for bit against the literal NumPy sampler (oracle.corr_np) given the same pyramid, for
    radius 0-5 x every grid of cases.LOOKUP_GRIDS x grid / jitter / edge coordinates.  plant(pyr) may write non-finite
    cells into the pyramid first; NaN then has to land on exactly the sampler's NaN positions.  Returns the number of
    cases."""
    n = 0
    for levels, grids in cases.LOOKUP_GRIDS.items():
        for b, h, w in grids:
            pyr = _oracle_pyramid(b, h, w, levels)
            if plant is not None:
                plant(pyr)
            pyr_dev = [dev(p) for p in pyr]
            for r in RADII:
                ocb = corr_np.CorrBlock.__new__(corr_np.CorrBlock)
                ocb.corr_pyramid, ocb.num_levels, ocb.radius = pyr, levels, r
                for kind in KINDS:
                    coords = cases.lookup_coords(b, h, w, kind)
                    got = _retrieve(T, pyr_dev, coords, r).cpu().numpy()
                    with np.errstate(invalid='ignore'):
                        want = ocb.retrieve(coords)
                    if not np.array_equal(got, want, equal_nan=True):
                        bad = (got != want) & ~(np.isnan(got) & np.isnan(want))
                        raise AssertionError(f'radius {r}, {levels} levels, grid {b}x{h}x{w}, {kind}: {int(bad.sum())} of '
                                             f'{bad.size} values differ, max-abs {float(np.abs(got - want).max()):.3e}')
                    n += 1
    return n


def lookup_kernel_names(T, radius, levels, grid):
    """Names of the lookup kernels one CorrBlock.retrieve launches (from the CUDA profiler).

    The library's launch counter says how many kernels the call launched (retrieve launches lookup kernels only).  The
    profiler receives kernel records from CUPTI asynchronously, and a capture can come back without some of them; such
    a capture says nothing about which kernel ran, so it is taken again, up to three times.  What it returns is only
    ever the names of kernels the profiler saw."""
    from torch.profiler import ProfilerActivity, profile
    from tf_raft_b200 import _lib
    b, h, w = grid
    pyr_dev = [dev(p) for p in _oracle_pyramid(b, h, w, levels)]
    coords = cases.lookup_coords(b, h, w, 'jitter')
    for _ in range(3):
        torch.cuda.synchronize()
        _lib.launch_count_reset()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _retrieve(T, pyr_dev, coords, radius)
            torch.cuda.synchronize()
        launched = _lib.launch_count()
        seen = [e for e in prof.key_averages() if 'lookup' in e.key]
        if sum(e.count for e in seen) >= launched:
            break
    return sorted({e.key for e in seen})


# The window kernel's configurations, vector and scalar loads, and one configuration of the generic kernel.
_KERNEL_PROBES = ((4, 4, (1, 8, 32)), (3, 4, (1, 8, 32)), (3, 4, (2, 9, 13)), (4, 4, (2, 9, 13)), (2, 5, (1, 17, 19)))


def test_lookup_bit_exact_every_radius_and_depth(T):
    for r, levels, grid in _KERNEL_PROBES:
        names = lookup_kernel_names(T, r, levels, grid)
        win = levels == 4 and r in (3, 4)
        assert len(names) == 1 and ('corr_lookup_win_kernel' in names[0]) == win, (r, levels, grid, names)
    assert lookup_forward_matrix(T) == len(RADII) * len(KINDS) * sum(len(g) for g in cases.LOOKUP_GRIDS.values())


_GATHER_SCRIPT = r'''
import os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], 'tests'))
import tf_raft_b200 as T
import test_gpu_geometry as g
for r, levels, grid in g._KERNEL_PROBES:
    print('KERNELS', r, levels, *g.lookup_kernel_names(T, r, levels, grid))
print('CHECKED', g.lookup_forward_matrix(T))
'''


def test_lookup_generic_kernel_bit_exact_at_the_window_configurations():
    """The same matrix with RAFT_B200_LOOKUP_GATHER=1, which sends every lookup to the generic kernel, (4, 4) and (3, 4)
    included.  The switch is read once per process, hence the subprocess."""
    res = subprocess.run([sys.executable, '-c', _GATHER_SCRIPT, ROOT], capture_output=True, text=True, timeout=600,
                         env={**os.environ, 'RAFT_B200_LOOKUP_GATHER': '1', 'PYTHONDONTWRITEBYTECODE': '1'})
    assert res.returncode == 0, res.stderr[-3000:]
    lines = res.stdout.splitlines()
    kernels = [l.split()[3:] for l in lines if l.startswith('KERNELS')]
    assert len(kernels) == len(_KERNEL_PROBES), res.stdout[-2000:]
    assert all(len(k) == 1 and 'corr_lookup_win_kernel' not in k[0] for k in kernels), kernels
    n = len(RADII) * len(KINDS) * sum(len(g) for g in cases.LOOKUP_GRIDS.values())
    assert f'CHECKED {n}' in lines, res.stdout[-2000:]


def _oracle_lookup_grads(pyr, coords, g, radius, dtype):
    P = [torch.from_numpy(p).to(dtype).requires_grad_(True) for p in pyr]
    c = torch.from_numpy(coords).to(dtype).requires_grad_(True)
    cb = rt.CorrBlock.__new__(rt.CorrBlock)
    cb.corr_pyramid, cb.num_levels, cb.radius = P, len(P), radius
    cb.retrieve(c).backward(torch.from_numpy(g).to(dtype))
    return c.grad, [q.grad for q in P]


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('radius,levels', [(3, 4), (4, 4), (2, 1), (4, 5), (0, 2), (5, 6)])
def test_lookup_backward_vs_fp64_autograd(T, radius, levels, kind):
    """d/d coords and d/d pyramid of the lookup against torch.autograd of the oracle sampler in fp64 (floor, ceil and
    gather carry no gradient; clamp passes it inside [0, size - 1], borders included).  The 'edge' coordinates decide
    the clamp branch and the integer taps, whose bilinear weights are all zero.  The kernel scatters with atomics, so
    the comparison is to a tolerance, the one of tests/test_train.py."""
    from tf_raft_b200.train import _Lookup
    for b, h, w in cases.LOOKUP_GRIDS[levels]:
        pyr = _oracle_pyramid(b, h, w, levels)
        coords = cases.lookup_coords(b, h, w, kind)
        g = np.random.default_rng(5).standard_normal((b, h, w, levels * (2 * radius + 1) ** 2)).astype(np.float32)
        gc64, gp64 = _oracle_lookup_grads(pyr, coords, g, radius, F64)
        gc32, gp32 = _oracle_lookup_grads(pyr, coords, g, radius, torch.float32)
        pyr_gpu = [dev(p).requires_grad_(True) for p in pyr]
        c_gpu = dev(coords).requires_grad_(True)
        _Lookup.apply(c_gpu, radius, *pyr_gpu).backward(dev(g))
        print(f'r={radius} levels={levels} {b}x{h}x{w} {kind}: d/dcoords max-abs {maxabs(c_gpu.grad, gc64):.2e} '
              f'(fp32 oracle {maxabs(gc32, gc64):.2e}, |grad| up to {float(gc64.abs().max()):.1f}); d/dpyramid max-abs '
              f'{max(maxabs(a.grad, t) for a, t in zip(pyr_gpu, gp64)):.2e} '
              f'(fp32 oracle {max(maxabs(a, t) for a, t in zip(gp32, gp64)):.2e})')
        np.testing.assert_allclose(c_gpu.grad.cpu().numpy(), gc64.numpy(), atol=2e-4, rtol=1e-4)
        for l in range(levels):
            np.testing.assert_allclose(pyr_gpu[l].grad.cpu().numpy(), gp64[l].numpy(), atol=1e-5, rtol=1e-5,
                                       err_msg=f'level {l}')


# --------------------------------------------------------------------------------------------- 4. encoders
@pytest.mark.parametrize('size', [(70, 98), (36, 52)], ids=_grid_id)
@pytest.mark.parametrize('norm', ['instance', 'batch', None])
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_encoder_odd_intermediate_sizes(T, variant, norm, size):
    """Native encoders on images that are not multiples of 8: the stride-2 stages see odd sizes (70 x 98: 35 x 49, then
    18 x 25, then 9 x 13; 36 x 52: 18 x 26, 9 x 13, then 5 x 7), so Keras 'same' padding is asymmetric there.  BatchNorm
    runs in training mode (batch statistics), the image is given raw (0..255) and normalised."""
    from tf_raft_b200.layers.extractor import BasicEncoder, SmallEncoder
    H, W = size
    out_dim = 256 if variant == 'raft' else 128
    p = cases.encoder_params(variant, norm, out_dim, seed=99 + H)
    training = norm == 'batch'
    im, _ = cases.images(2, H, W, seed0=H + W)
    x = (2 * (torch.from_numpy(im) / 255.0) - 1.0).permute(0, 3, 1, 2)
    truth = nhwc(rt.encoder(rt.Ops(p, F64), x.double(), 'enc', norm, training))
    fp32 = nhwc(rt.encoder(rt.Ops(p), x, 'enc', norm, training))
    assert tuple(truth.shape) == (2, -(-H // 8), -(-W // 8), out_dim)
    cls = BasicEncoder if variant == 'raft' else SmallEncoder
    for raw in (True, False):
        enc = cls(output_dim=out_dim, norm_type=norm, backend='native')
        enc.load_params(p, 'enc.')
        got = enc(dev(im) if raw else dev(x.permute(0, 2, 3, 1)), training=training, raw_image=raw)
        assert tuple(got.shape) == tuple(truth.shape)
        e = maxabs(got, truth)
        print(f'{variant} encoder, norm {norm}, {H}x{W}, raw_image={raw}: max-abs {e:.2e} '
              f'(fp32 oracle {maxabs(fp32, truth):.2e}), |out| up to {float(truth.abs().max()):.2f}')
        assert e < 2e-4


# --------------------------------------------------------------------------------------------- 5. the fused loop
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('grid', [(9, 128), (13, 11)], ids=_grid_id)
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_fused_loop_equals_the_public_ops(T, variant, grid, precision):
    """raft_b200_forward_loop (window lookup writing fp16 hi/lo operands with the convf1 im2col rider, fused
    coords1 += delta, mask head skipped where no prediction is asked for) must give, byte for byte, what the loop spelled
    out with CorrBlock.retrieve, update_block and upsample_flow gives, at every iteration and with last_only=True.
    Batch 2, on the 128 x 1 tile grid (TH = 1) and on a ragged 16 x 8 tile grid."""
    h, w = grid
    iters, bs = 3, 2
    p = weights.init_params(variant, 1234, bias_scale=0.05, norm_jitter=0.1)
    im1, im2 = cases.images(bs, 8 * h, 8 * w, 3, 4)
    a, b = dev(im1), dev(im2)
    model = (T.RAFT if variant == 'raft' else T.SmallRAFT)(iters=iters, iters_pred=iters, precision=precision)
    model.load_params(p)
    fmap1, fmap2, net, inp = model._encode(a, b, False)
    cb = T.CorrBlock(fmap1, fmap2, model.corr_levels, model.corr_radius, precision=precision)
    coords1 = T.coords_grid(bs, h, w)
    grid0 = coords1.clone()
    ups = []
    for _ in range(iters):
        corr = cb.retrieve(coords1)
        net, mask, delta = model.update_block([net, inp, corr, coords1 - grid0])
        coords1 = coords1 + delta
        ups.append(model.upsample_flow(coords1 - grid0, mask))
    full = model([a, b], training=False)
    assert len(full) == iters
    for i in range(iters):
        assert torch.equal(full[i], ups[i]), f'iteration {i}: max-abs {maxabs(full[i], ups[i]):.3e}'
    last = model([a, b], training=False, last_only=True)
    assert len(last) == 1 and torch.equal(last[0], ups[-1]), 'last_only differs from the loop spelled out'
