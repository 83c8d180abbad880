"""The correlation pyramid, the lookup and the fused loop on grids whose pyramid holds 2^31 elements or more.

corr_lookup_win_kernel addresses the pyramid with 32-bit offsets, so the host sends every lookup whose level 0 holds 2^31
elements or more (B*h*w query planes of h*w elements: 1728 x 1728 images at batch 1, or the Sintel grid at batch 42) to
the generic corr_lookup_kernel, and in raft_b200_forward_loop adds a separate flow_im2col_kernel launch for the convf1
planes the window kernel would have written.  The cases of cases.LARGE_CASES sit on both sides of that limit and one past
2^32, where every kernel on the path must address the pyramid with 64-bit offsets.

Each case needs 11 to 23 GB of device memory.  One case is alive at a time: a test releases it before the next starts,
and skips, naming both numbers, when the device has less free memory than the case needs plus 4 GB.  Only the planes of
the sampled queries (cases.large_sample) are copied back and compared with float64 references (pyramid, lookup
gradients) or the literal NumPy sampler (lookup forward, bit for bit).
"""
import gc
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import cases
from oracle import corr_np, raft_torch as rt, weights

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
GB = 1e9
HEADROOM = 4 * 10 ** 9
KINDS = ('grid', 'jitter', 'edge')
LEVELS, C = 4, 256
_PEAK = [0]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _grid_id(g):
    return 'x'.join(map(str, g))


def pyramid_bytes(B, h, w, levels=LEVELS):
    return sum(B * h * w * lh * lw * 4 for lh, lw in cases.level_sizes(h, w, levels))


def require_free(nbytes):
    """Skip unless the device has nbytes plus HEADROOM free."""
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + HEADROOM:
        pytest.skip(f'needs {nbytes / GB:.1f} GB of device memory plus {HEADROOM / GB:.0f} GB headroom; '
                    f'{free / GB:.1f} GB free')


def _release():
    # A failed test's traceback (kept for post-mortem debugging) holds its frames and with them its device tensors.
    sys.last_type = sys.last_value = sys.last_traceback = None
    if hasattr(sys, 'last_exc'):
        sys.last_exc = None
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope='module')
def T():
    import tf_raft_b200
    from tf_raft_b200 import _lib
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    yield tf_raft_b200
    print(f'\npeak device memory of the module: {_PEAK[0] / GB:.2f} GB ({torch.cuda.get_device_name()})')


@pytest.fixture(autouse=True)
def one_case_at_a_time():
    """Every test starts and ends with its large buffers released; prints its peak device memory."""
    _release()
    torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated()
    _PEAK[0] = max(_PEAK[0], peak)
    print(f'  peak device memory {peak / GB:.2f} GB')
    _release()


def _sample(B, h, w):
    qs = cases.large_sample(B, h, w)
    return qs, torch.from_numpy(qs).cuda()


def kernel_names(fn):
    """Names of the CUDA kernels fn() launches (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sorted({e.key for e in prof.key_averages()})


def lookup_kernels(names):
    return [n for n in names if 'corr_lookup' in n]


def check_lookup_kernel(names, path):
    """names (one lookup's kernels) ran the kernel cases.lookup_path predicts."""
    found = lookup_kernels(names)
    assert len(found) == 1, names
    if path == 'generic':
        assert 'corr_lookup_kernel' in found[0], found
    else:
        m = re.search(r'corr_lookup_win_kernel<\d+,\d+,(true|false),(true|false)>', found[0].replace(' ', ''))
        assert m and m.group(1) == ('true' if path == 'window-vec' else 'false'), found


# --------------------------------------------------------------------------------------------- 1. pyramid
PYRAMID_RUNS = [(c, 'f16x2') for c in cases.LARGE_CASES] + [((1, 216, 216), 'fp32'), ((1, 257, 256), 'fp32')]


@pytest.mark.parametrize('case,precision', PYRAMID_RUNS, ids=[f'{_grid_id(c)}-{p}' for c, p in PYRAMID_RUNS])
def test_pyramid_rows_vs_fp64(T, case, precision):
    """Every level of the sampled queries' planes against the fp64 volume pooled the reference's way, with the
    tolerance of test_corr_pyramid_vs_fp64.  The fp32 build's level 0 is the only place corr_fp32_kernel writes past
    2^31 and 2^32; the f16x2 build writes it from corr_tc_kernel's store."""
    B, h, w = case
    require_free(pyramid_bytes(B, h, w) + 6 * B * h * w * C * 4)
    qs, idx = _sample(B, h, w)
    f1, f2 = cases.fmaps(B, h, w, C)
    truth = cases.corr_rows(f1, f2, qs, LEVELS)
    cb = T.CorrBlock(dev(f1), dev(f2), num_levels=LEVELS, radius=4, precision=precision)
    del f1, f2
    got = [p[idx].cpu() for p in cb.corr_pyramid]
    del cb
    for l, (lh, lw) in enumerate(cases.level_sizes(h, w, LEVELS)):
        assert tuple(got[l].shape) == (len(qs), lh, lw, 1)
        err = (got[l].double() - truth[l]).abs()
        worst = int(err.reshape(len(qs), -1).amax(1).argmax())
        print(f'{precision} {_grid_id(case)} level {l} ({lh}x{lw}): max-abs {float(err.max()):.2e} at query '
              f'{int(qs[worst])} (tolerance 2e-5 + 2e-5 |x|), |corr| up to {float(truth[l].abs().max()):.2f}, '
              f'{len(qs)} queries')
        np.testing.assert_allclose(got[l].numpy(), truth[l].numpy(), atol=2e-5, rtol=2e-5, err_msg=f'level {l}')


# --------------------------------------------------------------------------------------------- 2. lookup forward
@pytest.mark.parametrize('case', cases.LARGE_CASES, ids=_grid_id)
def test_lookup_rows_bit_exact(T, case):
    """CorrBlock.retrieve (radius 4) over the whole grid; the sampled queries' rows bit for bit against the NumPy
    sampler applied to the GPU's own planes of those queries (the sampler reads only the query's planes)."""
    B, h, w = case
    nch = LEVELS * 81
    require_free(pyramid_bytes(B, h, w) + 4 * B * h * w * C * 4 + 2 * B * h * w * nch * 4)
    qs, idx = _sample(B, h, w)
    f1, f2 = cases.fmaps(B, h, w, C)
    cb = T.CorrBlock(dev(f1), dev(f2), num_levels=LEVELS, radius=4, precision='f16x2')
    del f1, f2
    ocb = corr_np.CorrBlock.__new__(corr_np.CorrBlock)
    ocb.corr_pyramid, ocb.num_levels, ocb.radius = [p[idx].cpu().numpy() for p in cb.corr_pyramid], LEVELS, 4
    for kind in KINDS:
        coords = cases.lookup_coords(B, h, w, kind)
        c = dev(coords)
        got = cb.retrieve(c).reshape(-1, nch)[idx].cpu().numpy()
        want = ocb.retrieve(coords.reshape(-1, 2)[qs].reshape(1, len(qs), 1, 2)).reshape(len(qs), nch)
        if not np.array_equal(got, want):
            bad = np.nonzero((got != want).any(1))[0]
            raise AssertionError(f'{_grid_id(case)} {kind}: {len(bad)} of {len(qs)} sampled rows differ (queries '
                                 f'{qs[bad][:8].tolist()}), max-abs {float(np.abs(got - want).max()):.3e}')


_KERNEL_SCRIPT = r'''
import os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], 'tests'))
import torch
import cases
import tf_raft_b200 as T
import test_gpu_large as L
for B, h, w in cases.LARGE_CASES:
    cb = T.CorrBlock.__new__(T.CorrBlock)
    cb.corr_pyramid = [torch.zeros((B * h * w, lh, lw, 1), device='cuda') for lh, lw in cases.level_sizes(h, w, 4)]
    cb.num_levels, cb.radius, cb._shape = 4, 4, (B, h, w)
    c = L.dev(cases.lookup_coords(B, h, w, 'jitter'))
    print('KERNELS', B, h, w, '|'.join(n.replace(' ', '') for n in L.kernel_names(lambda: cb.retrieve(c))), flush=True)
    del cb, c
    torch.cuda.empty_cache()
'''


def test_lookup_kernel_on_each_side_of_the_limit():
    """Which lookup kernel CorrBlock.retrieve runs on each large grid (torch.profiler): the one cases.lookup_path
    predicts.  The choice depends on the shapes only, so the pyramid is zeros.  It runs in a fresh process: late in a
    long test session the profiler has been seen to return the launch of a lone kernel without the kernel itself."""
    B, h, w = max(cases.LARGE_CASES, key=lambda c: pyramid_bytes(*c))
    require_free(pyramid_bytes(B, h, w) + 2 * 10 ** 9)
    res = subprocess.run([sys.executable, '-c', _KERNEL_SCRIPT, ROOT], capture_output=True, text=True, timeout=600,
                         env={**os.environ, 'PYTHONDONTWRITEBYTECODE': '1'})
    assert res.returncode == 0, res.stderr[-3000:]
    lines = [l.split() for l in res.stdout.splitlines() if l.startswith('KERNELS')]
    assert len(lines) == len(cases.LARGE_CASES), res.stdout[-2000:]
    for _, B, h, w, names in lines:
        path = cases.lookup_path(int(B), int(h), int(w), LEVELS, 4, LEVELS * 81)
        print(f'{B}x{h}x{w}: {path}, ran {lookup_kernels(names.split("|"))}')
        check_lookup_kernel(names.split('|'), path)


# --------------------------------------------------------------------------------------------- 3. lookup backward
def test_lookup_backward_past_2_31(T):
    """d/d coords and d/d pyramid of the lookup at 216 x 216 (level 0 past 2^31 elements) with a gradient that is zero
    except on the sampled queries: their planes and coordinates against torch.autograd of the oracle sampler in fp64
    (the tolerances of test_lookup_backward_vs_fp64_autograd), every other plane and coordinate exactly zero."""
    from tf_raft_b200.train import _Lookup
    B, h, w = 1, 216, 216
    nq, nch = B * h * w, LEVELS * 81
    require_free(2 * pyramid_bytes(B, h, w) + 4 * nq * C * 4 + 4 * nq * nch * 4)
    qs, idx = _sample(B, h, w)
    f1, f2 = cases.fmaps(B, h, w, C)
    pyr = T.CorrBlock(dev(f1), dev(f2), num_levels=LEVELS, radius=4, precision='f16x2').corr_pyramid
    del f1, f2
    planes = [p[idx].cpu().double() for p in pyr]
    for p in pyr:
        p.requires_grad_(True)
    for kind in KINDS:
        coords = cases.lookup_coords(B, h, w, kind).reshape(nq, 2)
        g = np.zeros((nq, nch), np.float32)
        g[qs] = np.random.default_rng(5).standard_normal((len(qs), nch))
        c_gpu = dev(coords.reshape(B, h, w, 2)).requires_grad_(True)
        _Lookup.apply(c_gpu, 4, *pyr).backward(dev(g.reshape(B, h, w, nch)))

        P = [x.clone().requires_grad_(True) for x in planes]
        c64 = torch.from_numpy(coords[qs]).double().reshape(1, len(qs), 1, 2).requires_grad_(True)
        ocb = rt.CorrBlock.__new__(rt.CorrBlock)
        ocb.corr_pyramid, ocb.num_levels, ocb.radius = P, LEVELS, 4
        ocb.retrieve(c64).backward(torch.from_numpy(g[qs]).double().reshape(1, len(qs), 1, nch))

        gc_rows = c_gpu.grad.reshape(nq, 2)[idx].cpu()
        gp_rows = [p.grad[idx].cpu() for p in pyr]
        print(f'{kind}: d/dcoords max-abs {float((gc_rows.double() - c64.grad.reshape(-1, 2)).abs().max()):.2e}, '
              f'd/dpyramid max-abs {max(float((a.double() - b.grad).abs().max()) for a, b in zip(gp_rows, P)):.2e}')
        np.testing.assert_allclose(gc_rows.numpy(), c64.grad.reshape(-1, 2).numpy(), atol=2e-4, rtol=1e-4)
        for l in range(LEVELS):
            np.testing.assert_allclose(gp_rows[l].numpy(), P[l].grad.numpy(), atol=1e-5, rtol=1e-5, err_msg=f'level {l}')
        # nothing outside the sampled queries: count on the device, a slice of rows at a time (no copy of a level)
        for l, p in enumerate(pyr):
            total = sum(int(torch.count_nonzero(p.grad[i:i + 4096])) for i in range(0, nq, 4096))
            assert total == int(torch.count_nonzero(gp_rows[l])), f'level {l}: gradient outside the sampled planes'
            p.grad = None
        assert int(torch.count_nonzero(c_gpu.grad)) == int(torch.count_nonzero(gc_rows)), 'd/dcoords outside the sample'
        del c_gpu


# --------------------------------------------------------------------------------------------- 4. the fused loop
def loop_kernels(model, a, b, **kw):
    """Lookup and flow im2col kernels a model([a, b]) call launches."""
    def call():
        model([a, b], training=False, **kw)
        model._last = None                 # holds the call's pyramid: one alive at a time
    names = kernel_names(call)
    return [n for n in names if 'corr_lookup' in n or 'flow_im2col' in n]


def check_loop_kernels(names, path, precision):
    """The loop ran the lookup kernel cases.lookup_path predicts, and (tensor-core path) flow_im2col_kernel exactly when
    that lookup is the generic kernel: the window kernel writes the convf1 planes itself."""
    win = [n for n in names if 'corr_lookup_win_kernel' in n]
    gen = [n for n in names if 'corr_lookup_kernel' in n]
    im2col = [n for n in names if 'flow_im2col_kernel' in n]
    assert (bool(win), bool(gen)) == ((False, True) if path == 'generic' else (True, False)), names
    if precision == 'f16x2':
        assert bool(im2col) == (path == 'generic'), names


@pytest.mark.parametrize('precision', ('f16x2', 'fp32'))
@pytest.mark.parametrize('grid', [(215, 215), (216, 216)], ids=_grid_id)
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_fused_loop_equals_the_public_ops_at_the_limit(T, variant, grid, precision):
    """test_fused_loop_equals_the_public_ops on 1720 x 1720 images (window lookup, im2col rider) and on 1728 x 1728
    (generic lookup writing the fp16 operand planes, separate flow_im2col_kernel launch), batch 1, 2 iterations: the
    loop gives, byte for byte, what the loop spelled out with CorrBlock.retrieve, update_block and upsample_flow gives,
    at every iteration and with last_only=True."""
    h, w = grid
    iters, bs = 2, 1
    require_free(pyramid_bytes(bs, h, w) + 6 * 10 ** 9)
    p = weights.init_params(variant, 1234, bias_scale=0.05, norm_jitter=0.1)
    im1, im2 = cases.images(bs, 8 * h, 8 * w, 3, 4)
    a, b = dev(im1), dev(im2)
    model = (T.RAFT if variant == 'raft' else T.SmallRAFT)(iters=iters, iters_pred=iters, precision=precision)
    model.load_params(p)
    fmap1, fmap2, net, inp = model._encode(a, b, False)
    cb = T.CorrBlock(fmap1, fmap2, model.corr_levels, model.corr_radius, precision=precision)
    del fmap1, fmap2
    coords1 = T.coords_grid(bs, h, w)
    grid0 = coords1.clone()
    ups = []
    for _ in range(iters):
        corr = cb.retrieve(coords1)
        net, mask, delta = model.update_block([net, inp, corr, coords1 - grid0])
        coords1 = coords1 + delta
        ups.append(model.upsample_flow(coords1 - grid0, mask))
    del cb, corr
    _release()

    stride = (384 if variant == 'raft' else 256) if precision == 'f16x2' else model.corr_levels * (2 * model.corr_radius + 1) ** 2
    path = cases.lookup_path(bs, h, w, model.corr_levels, model.corr_radius, stride)
    names = loop_kernels(model, a, b, last_only=True)
    print(f'{variant} {precision} {_grid_id(grid)}: {path}, the loop ran {names}')
    check_loop_kernels(names, path, precision)
    _release()

    full = model([a, b], training=False)
    model._last = None
    assert len(full) == iters
    for i in range(iters):
        assert torch.equal(full[i], ups[i]), f'iteration {i}: max-abs {float((full[i] - ups[i]).abs().max()):.3e}'
    del full
    _release()
    last = model([a, b], training=False, last_only=True)
    model._last = None
    assert len(last) == 1 and torch.equal(last[0], ups[-1]), 'last_only differs from the loop spelled out'


_GATHER_LOOP_SCRIPT = r'''
import os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], 'tests'))
import cases
import tf_raft_b200 as T
from oracle import weights
import test_gpu_geometry as g
import test_gpu_large as L
for variant in ('raft', 'small'):
    for h, w in ((9, 128), (13, 11)):
        for precision in g.PRECISIONS:
            g.test_fused_loop_equals_the_public_ops(T, variant, (h, w), precision)
            model = (T.RAFT if variant == 'raft' else T.SmallRAFT)(iters=2, iters_pred=2, precision=precision)
            model.load_params(weights.init_params(variant, 1234, bias_scale=0.05, norm_jitter=0.1))
            im1, im2 = cases.images(2, 8 * h, 8 * w, 3, 4)
            names = L.loop_kernels(model, L.dev(im1), L.dev(im2))
            print('EQUAL', variant, h, w, precision, '|'.join(n.replace(' ', '') for n in names))
'''


def test_fused_loop_equals_the_public_ops_on_the_generic_lookup():
    """test_fused_loop_equals_the_public_ops with RAFT_B200_LOOKUP_GATHER=1, which sends every lookup to the generic
    kernel: the loop then takes the path of grids past the window kernel's limit (the generic kernel writes the fp16
    operand planes, flow_im2col_kernel writes the convf1 planes) at small sizes.  The switch is read once per process,
    hence the subprocess."""
    res = subprocess.run([sys.executable, '-c', _GATHER_LOOP_SCRIPT, ROOT], capture_output=True, text=True, timeout=600,
                         env={**os.environ, 'RAFT_B200_LOOKUP_GATHER': '1', 'PYTHONDONTWRITEBYTECODE': '1'})
    assert res.returncode == 0, res.stderr[-3000:]
    lines = [l.split() for l in res.stdout.splitlines() if l.startswith('EQUAL')]
    assert len(lines) == 8, res.stdout[-2000:]
    for *_, precision, names in lines:
        check_loop_kernels(names.split('|'), 'generic', precision)
    print('\n'.join(' '.join(l) for l in lines))
