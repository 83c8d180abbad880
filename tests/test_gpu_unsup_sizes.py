"""raft_b200_unsup_loss_norm where kernels go wrong, against the closed-form float64 restatement
(oracle/unsup_np.py, direction_closed_form): the training shapes (a 1024-CTA grid-stride loop), multi-megapixel and
ragged shapes, the 7 x 7 frame with one masked pixel, empty masks and the 2 x 2 minimum; every grid the host can pick,
up to the 1056-CTA cap; the parameter edges; a caller-supplied census normaliser; and a frame past 2^31 census
elements.

Each case calls the entry point directly for one direction (target census, source census, target image, occlusion,
n predictions) and checks the loss terms sums[0..3] (the mask count exact, the rest within 1e-5 relative) and every
gradient element (within `grad_tol` of the largest).  The oracle is fed gamma rounded to float32, as the kernel
receives it."""
import gc
import math
import sys

import numpy as np
import pytest
import torch

from oracle import unsup_np
from test_gpu_unsup import _flows, _texture

pytestmark = pytest.mark.gpu
F32 = np.float32
GB = 1e9
HEADROOM = 4 * 10 ** 9
NPARTIALS = 4096                     # train._UnsupLoss.NPARTIALS: a grid of up to 1024 CTAs


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def grad_tol(h, w):
    """Gradient bound relative to the largest entry.  The kernel takes the bilinear weight ax = px - floor(px) from the
    float32 landing px = x + F_x, which carries the rounding of px, up to 2^-24 max(H, W); the oracle's ax is exact.
    Measured on an H100: 2.5e-6 at 24 x 40, 1.7e-5 at 64 x 96, 9.3e-5 at 368 x 496, 5.4e-4 at 1080 x 2560, about
    2e-7 max(H, W) throughout; landings on texels (ax = 0) stay below 4e-7 at every size."""
    return 1e-5 + 8 * 2.0 ** -24 * max(h, w)


def _call(ct, cs, img, occ, flows, cw=1.0, sw=0.5, ew=150.0, gamma=0.8, npartials=NPARTIALS, norm=None,
          partials=None):
    """One raft_b200_unsup_loss_norm call on device tensors -> (sums (4,) float64 NumPy, grad (n, B, H, W, 2) on the
    device)."""
    from tf_raft_b200 import _lib
    n, b, h, w, _ = flows.shape
    grad = torch.empty_like(flows)
    if partials is None:
        partials = torch.empty(npartials, dtype=torch.float64, device='cuda')
    sums = torch.empty(4, dtype=torch.float64, device='cuda')
    _lib.call('unsup_loss_norm', flows.device, _lib.ptr(ct), _lib.ptr(cs), _lib.ptr(img), _lib.ptr(occ),
              _lib.ptr(flows), n, b, h, w, cw, sw, ew, gamma, _lib.ptr(partials), npartials, _lib.ptr(sums),
              _lib.ptr(grad), _lib.ptr(norm))
    return sums.cpu().numpy(), grad


def _inputs(b, h, w, n, case='random', seed=0, occ_p=0.25, images=None):
    rng = np.random.default_rng(seed)
    im_t, im_s = images if images is not None else (_texture(b, h, w, seed + 1), _texture(b, h, w, seed + 2))
    occ = (rng.random((b, h, w)) < occ_p).astype(np.uint8)
    flows = np.stack(_flows(case, n, b, h, w, rng))
    return im_t, im_s, occ, flows


def _run(im_t, im_s, occ, flows, cw=1.0, sw=0.5, ew=150.0, gamma=0.8, norm=None, **kw):
    """The kernel and the oracle on the same direction -> (sums, grad as NumPy, oracle (lc, ls, count, grads))."""
    from tf_raft_b200.losses import census_transform
    ct_d, cs_d = census_transform(dev(im_t)), census_transform(dev(im_s))
    norm_d = None if norm is None else torch.tensor([norm], dtype=torch.float64, device='cuda')
    sums, grad = _call(ct_d, cs_d, dev(im_t), dev(occ), dev(flows), cw, sw, ew, gamma, norm=norm_d, **kw)
    b, h, w = occ.shape
    mask = unsup_np.border_mask(b, h, w) & (occ == 0)
    want = unsup_np.direction_closed_form(unsup_np.census(im_t), unsup_np.census(im_s), im_t, mask, list(flows), cw, sw,
                                          ew, float(F32(gamma)), norm)
    return sums, grad.cpu().numpy(), want


def _check(sums, grad, want, cw=1.0, sw=0.5, what=''):
    """sums against (L_c, L_s, count, share), every gradient element against the oracle's; -> (worst loss error,
    worst gradient error / largest entry)."""
    lc, ls, count, want_g = want
    assert sums[2] == count, f'{what}: mask count {sums[2]} != {count}'
    worst = 0.0
    for k, v in ((0, lc), (1, ls), (3, cw / 2 * lc + sw / 2 * ls)):
        if math.isnan(v):
            assert math.isnan(sums[k]), f'{what}: sums[{k}] = {sums[k]}, oracle NaN'
            continue
        assert sums[k] == pytest.approx(v, rel=1e-5, abs=1e-30), f'{what}: sums[{k}] = {sums[k]!r}, oracle {v!r}'
        if v != 0:
            worst = max(worst, abs(sums[k] - v) / abs(v))
    want_g = np.stack(want_g)
    finite = np.isfinite(want_g)
    np.testing.assert_array_equal(np.isnan(grad), np.isnan(want_g), err_msg=f'{what}: NaN pattern')
    np.testing.assert_array_equal(np.isinf(grad), np.isinf(want_g), err_msg=f'{what}: inf pattern')
    scale = float(np.abs(want_g[finite]).max(initial=0.0))
    err = float(np.abs(grad[finite] - want_g[finite]).max(initial=0.0))
    assert err <= grad_tol(*grad.shape[2:4]) * scale, f'{what}: gradient error {err:.3e}, largest entry {scale:.3e}'
    return worst, err / scale if scale else 0.0


# --------------------------------------------------------------------------------------------- shapes
TRAINING = [(4, 368, 496, 12), (2, 400, 720, 12)]
KINDS = ['random', 'integer', 'leaving', 'flat', 'nonfinite']
OTHER = [(1, 1080, 2560, 2), (5, 37, 53, 4), (3, 7, 7, 2), (2, 6, 40, 3), (2, 40, 6, 3), (1, 2, 2, 1)]


def _grid(b, h, w, npartials=NPARTIALS):
    return min(npartials // 4, -(-b * h * w // 256), 1056)


@pytest.mark.parametrize('shape,case', [(s, k) for s in TRAINING for k in KINDS] + [(s, 'random') for s in OTHER],
                         ids=lambda v: 'x'.join(map(str, v)) if isinstance(v, tuple) else v)
def test_loss_and_gradient_at_every_shape(shape, case):
    b, h, w, n = shape
    images = None
    if case == 'flat':
        images = (_texture(b, h, w, 1), _texture(b, h, w, 2))
        images[0][:, :, : w // 3] = 128.0                                   # zero image differences: edge weight 1
    im_t, im_s, occ, flows = _inputs(b, h, w, n, case, seed=sum(shape) + len(case), images=images,
                                     occ_p=0.0 if h == w == 7 else 0.25)
    grid = _grid(b, h, w)
    if shape == (4, 368, 496, 12):
        assert grid == 1024 and b * h * w > 2.7 * grid * 256                # every thread walks the loop ~2.8 times
    if shape == (5, 37, 53, 4):
        assert b * h * w - (grid - 1) * 256 == 77                           # 77 live threads in the last CTA
    sums, grad, want = _run(im_t, im_s, occ, flows)
    if h == w == 7:
        assert want[2] == b                                                 # one masked pixel, (3, 3), per image
    if min(h, w) < 7:
        assert want[2] == 0 and sums[0] == 0.0
    worst_loss, worst_grad = _check(sums, grad, want, what=f'{shape} {case}')
    print(f'{shape} {case}: grid {grid}, count {int(sums[2])}, worst loss error {worst_loss:.2e} relative, worst '
          f'gradient error {worst_grad:.2e} of the largest')


# --------------------------------------------------------------------------------------------- grids
def test_every_grid_gives_the_same_gradient_bits():
    """npartials 4 .. 16384: grids of 1, 2, 3, 129, 1024, 1056 (the cap) and 1056 CTAs.  The gradient depends on the
    grid through nothing (the mask count is an exact integer), so it is bit-identical; the loss sums in another order
    and agrees to 1e-13; each matches the oracle; the call writes partials [0, 4 * grid) and nothing past it."""
    from tf_raft_b200.losses import census_transform
    b, h, w, n = 4, 368, 496, 4
    im_t, im_s, occ, flows = _inputs(b, h, w, n, seed=7)
    ct, cs, img, occ_d, flows_d = census_transform(dev(im_t)), census_transform(dev(im_s)), dev(im_t), dev(occ), dev(flows)
    mask = unsup_np.border_mask(b, h, w) & (occ == 0)
    want = unsup_np.direction_closed_form(unsup_np.census(im_t), unsup_np.census(im_s), im_t, mask, list(flows),
                                          gamma=float(F32(0.8)))
    ref = None
    grids = []
    for npartials in (4, 8, 12, 516, 4096, 4224, 16384):
        grid = _grid(b, h, w, npartials)
        grids.append(grid)
        partials = torch.full((npartials,), float('nan'), dtype=torch.float64, device='cuda')
        sums, grad = _call(ct, cs, img, occ_d, flows_d, npartials=npartials, partials=partials)
        part = partials.cpu().numpy()
        assert np.isfinite(part[:4 * grid]).all(), f'npartials {npartials}: a partial of the grid left unwritten'
        assert np.isnan(part[4 * grid:]).all(), f'npartials {npartials}: written past 4 * grid = {4 * grid}'
        grad = grad.cpu().numpy()
        _check(sums, grad, want, what=f'npartials {npartials}')
        if ref is None:
            ref = (sums, grad)
            continue
        assert grad.tobytes() == ref[1].tobytes(), f'npartials {npartials}: gradient bits differ from grid 1'
        assert sums[2] == ref[0][2]
        for k in (0, 1, 3):
            assert sums[k] == pytest.approx(ref[0][k], rel=1e-13), (npartials, k, sums[k], ref[0][k])
    assert grids == [1, 2, 3, 129, 1024, 1056, 1056]


# --------------------------------------------------------------------------------------------- parameter edges
MID = (2, 64, 96, 3)


def test_every_pixel_occluded():
    """count 0: L_c and the census share exactly 0, and the gradient is that of census_weight 0 bit for bit."""
    b, h, w, n = MID
    im_t, im_s, _, flows = _inputs(b, h, w, n, seed=11)
    occ = np.ones((b, h, w), dtype=np.uint8)
    sums, grad, want = _run(im_t, im_s, occ, flows)
    _check(sums, grad, want, what='occ all ones')
    assert sums[2] == 0 and sums[0] == 0.0
    sums0, grad0, _ = _run(im_t, im_s, occ, flows, cw=0.0)
    assert sums[3] == sums0[3] and grad.tobytes() == grad0.tobytes()


def test_nothing_occluded():
    b, h, w, n = MID
    im_t, im_s, _, flows = _inputs(b, h, w, n, seed=12)
    sums, grad, want = _run(im_t, im_s, np.zeros((b, h, w), dtype=np.uint8), flows)
    assert sums[2] == b * (h - 6) * (w - 6)
    _check(sums, grad, want, what='occ all zeros')


@pytest.mark.parametrize('cw,sw', [(0.0, 0.5), (1.0, 0.0)], ids=['census_weight=0', 'smoothness_weight=0'])
def test_zero_weights(cw, sw):
    b, h, w, n = MID
    im_t, im_s, occ, flows = _inputs(b, h, w, n, seed=13)
    sums, grad, want = _run(im_t, im_s, occ, flows, cw=cw, sw=sw)
    _check(sums, grad, want, cw, sw, what=f'cw {cw} sw {sw}')
    assert sums[3] == (cw / 2 * sums[0] if sw == 0 else sw / 2 * sums[1])


def test_edge_weight_zero_makes_every_weight_one():
    b, h, w, n = MID
    im_t, im_s, occ, flows = _inputs(b, h, w, n, seed=14)
    sums, grad, want = _run(im_t, im_s, occ, flows, ew=0.0)
    _check(sums, grad, want, what='edge_weight 0')
    plain = unsup_np.direction_closed_form(unsup_np.census(im_t), unsup_np.census(im_s), np.zeros_like(im_t),
                                           np.zeros((b, h, w), dtype=bool), list(flows), gamma=float(F32(0.8)))
    assert sums[1] == pytest.approx(plain[1], rel=1e-5)                 # as if the image were flat


def test_edge_weight_1e4_underflows_every_weight():
    """On a checkerboard (neighbours differ by 255), exp(-1e4 ...) is 0: with census_weight 0 the gradient is exactly 0
    wherever all four pairs lie on the checkerboard, and the smoothness sum over those pairs vanishes."""
    b, h, w, n = MID
    im_t, im_s, occ, flows = _inputs(b, h, w, n, seed=15)
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing='ij')
    im_t[:, :, : w // 2] = (255.0 * ((xs + ys) % 2))[:, : w // 2, None]
    sums, grad, want = _run(im_t, im_s, occ, flows, ew=1e4)
    _check(sums, grad, want, what='edge_weight 1e4')
    sums0, grad0, want0 = _run(im_t, im_s, occ, flows, cw=0.0, ew=1e4)
    _check(sums0, grad0, want0, 0.0, what='edge_weight 1e4, census_weight 0')
    assert not grad0[:, :, :, : w // 2 - 1].any()
    assert grad0[:, :, :, w // 2 + 1:].any()
    im_t[:] = (255.0 * ((xs + ys) % 2))[..., None]                      # the whole frame: no smoothness at all
    sums1, grad1, _ = _run(im_t, im_s, occ, flows, cw=0.0, ew=1e4)
    assert sums1[1] == 0.0 and sums1[3] == 0.0 and not grad1.any()


@pytest.mark.parametrize('gamma', [0.0, 1.0, 1.25])
def test_gamma_edges(gamma):
    b, h, w, n = MID
    im_t, im_s, occ, flows = _inputs(b, h, w, n, seed=16)
    sums, grad, want = _run(im_t, im_s, occ, flows, gamma=gamma)
    _check(sums, grad, want, what=f'gamma {gamma}')
    if gamma == 0.0:                                                    # gamma^0 = 1 for the last prediction only
        assert not grad[:-1].any() and grad[-1].any()


def test_supplied_census_normaliser():
    """census_norm = 3 x the call's own count: L_c is a third of the NULL call's, the mask count is still the call's
    own, and both match the oracle given the same normaliser.  With NULL the call gives raft_b200_unsup_loss's bits."""
    from tf_raft_b200 import _lib
    from tf_raft_b200.losses import census_transform
    b, h, w, n = MID
    im_t, im_s, occ, flows = _inputs(b, h, w, n, seed=17)
    own, grad_own, want_own = _run(im_t, im_s, occ, flows)
    _check(own, grad_own, want_own, what='own count')
    img_d, occ_d, flows_d = dev(im_t), dev(occ), dev(flows)
    ct, cs = census_transform(img_d), census_transform(dev(im_s))
    grad_v2 = torch.empty_like(flows_d)
    part = torch.empty(NPARTIALS, dtype=torch.float64, device='cuda')
    sums_v2 = torch.empty(4, dtype=torch.float64, device='cuda')
    _lib.call('unsup_loss', flows_d.device, _lib.ptr(ct), _lib.ptr(cs), _lib.ptr(img_d), _lib.ptr(occ_d),
              _lib.ptr(flows_d), n, b, h, w, 1.0, 0.5, 150.0, 0.8, _lib.ptr(part), NPARTIALS, _lib.ptr(sums_v2),
              _lib.ptr(grad_v2))
    assert sums_v2.cpu().numpy().tobytes() == own.tobytes() and grad_v2.cpu().numpy().tobytes() == grad_own.tobytes()
    sums, grad, want = _run(im_t, im_s, occ, flows, norm=3.0 * own[2])
    _check(sums, grad, want, what='3 x own count')
    assert sums[2] == own[2] and sums[0] == pytest.approx(own[0] / 3, rel=1e-12)
    assert sums[1] == own[1]
    assert not np.array_equal(grad, grad_own)


# --------------------------------------------------------------------------------------------- past 2^31 census elements
def _release():
    sys.last_type = sys.last_value = sys.last_traceback = None
    if hasattr(sys, 'last_exc'):
        sys.last_exc = None
    gc.collect()
    torch.cuda.empty_cache()


def test_past_2_31_census_elements():
    """(6, 2160, 3840), n = 1: 2.39e9 census elements, so the pixel index times 48 passes 2^31 inside image 5.
    image2 = image1 (one census serves as target and source) and the flow is zero outside three row bands -- the first
    rows, the rows around census element 2^31 and the last rows -- so outside them D = 0 and every smoothness
    difference vanishes.  The band flows are integers, so every landing is on a texel and the gradient bound is the
    small frames' 1e-5 (fractional landings at x ~ 3800 carry float32 rounding of up to 1.2e-4 px, see grad_tol, which
    this case does not test).  The census of each band is checked bit for bit against NumPy; each band plus a 3-row
    margin then goes to the oracle with the frame's mask count and pair counts; the gradient must be exactly 0
    elsewhere."""
    from tf_raft_b200.losses import census_transform
    b, h, w = 6, 2160, 3840
    assert b * h * w * 48 >= 2 ** 31
    need = b * h * w * (48 * 4 + 3 * 4 + 2 * 2 * 4 + 1)                  # census, image, flow and gradient, occlusion
    _release()
    free, _ = torch.cuda.mem_get_info()
    if free < need + HEADROOM:
        pytest.skip(f'needs {need / GB:.1f} GB of device memory plus {HEADROOM / GB:.0f} GB headroom; '
                    f'{free / GB:.1f} GB free')
    torch.cuda.reset_peak_memory_stats()
    p31 = 2 ** 31 // 48
    b31, y31 = p31 // (h * w), p31 % (h * w) // w
    bands = [(0, 0, 8), (b31, y31 - 4, y31 + 5), (b - 1, h - 8, h)]
    gen = torch.Generator(device='cuda').manual_seed(5)
    img = torch.rand((b, 3, h, w), generator=gen, device='cuda') * 255.0
    # blurred as _texture blurs
    img = torch.nn.functional.avg_pool2d(torch.nn.functional.pad(img, (1, 1, 1, 1), mode='circular'), 3, stride=1)
    img = img.permute(0, 2, 3, 1).contiguous()
    census = census_transform(img)
    flows = torch.zeros((1, b, h, w, 2), device='cuda')
    occ = torch.zeros((b, h, w), dtype=torch.uint8, device='cuda')
    rng = np.random.default_rng(3)
    band_flows, band_occ = [], []
    for bi, r0, r1 in bands:
        # integer flows of at most 2 px: every landing on a texel within 2 rows, where the float32 landing is exact
        f = np.round(np.clip(rng.standard_normal((1, 1, r1 - r0, w, 2)) * 1.5, -2.0, 2.0)).astype(F32)
        o = (rng.random((1, r1 - r0, w)) < 0.25).astype(np.uint8)
        flows[:, bi:bi + 1, r0:r1] = dev(f)
        occ[bi:bi + 1, r0:r1] = dev(o)
        band_flows.append(f)
        band_occ.append(o)
    torch.cuda.synchronize()
    import time
    t0 = time.perf_counter()
    sums, grad = _call(census, census, img, occ, flows)
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated()
    border = unsup_np.border_mask(b, h, w)
    count = int(border.sum()) - sum(int((band_o.astype(bool) & border[bi:bi + 1, r0:r1]).sum())
                                    for (bi, r0, r1), band_o in zip(bands, band_occ))
    assert sums[2] == count
    pairs = (b * h * (w - 1), b * (h - 1) * w)
    lc = ls = 0.0
    band_count = 0
    worst = 0.0
    for (bi, r0, r1), f, o in zip(bands, band_flows, band_occ):
        s0, s1 = max(0, r0 - 3), min(h, r1 + 3)                            # the band plus a 3-row margin
        sub_img = img[bi:bi + 1, s0:s1].cpu().numpy()
        sub_census = census[bi:bi + 1, s0:s1].cpu().numpy()
        c0, c1 = max(0, s0 - 3), min(h, s1 + 3)                            # its census needs 3 more rows each side
        want_census = unsup_np.census(img[bi:bi + 1, c0:c1].cpu().numpy())[:, s0 - c0:s1 - c0]
        np.testing.assert_array_equal(sub_census, want_census, err_msg=f'census of rows {s0}..{s1} of image {bi}')
        mask = np.zeros((1, s1 - s0, w), dtype=bool)
        mask[:, r0 - s0:r1 - s0] = border[bi:bi + 1, r0:r1] & (o == 0)
        sub_flow = flows[0, bi:bi + 1, s0:s1].cpu().numpy()
        blc, bls, bcount, bgrad = unsup_np.direction_closed_form(sub_census, sub_census, sub_img, mask, [sub_flow],
                                                                 census_norm=max(count, 1), pairs=pairs,
                                                                 gamma=float(F32(0.8)))
        lc, ls, band_count = lc + blc, ls + bls, band_count + bcount
        got = grad[0, bi:bi + 1, s0:s1].cpu().numpy()
        scale = float(np.abs(bgrad[0]).max())
        err = float(np.abs(got - bgrad[0]).max())
        assert err <= 1e-5 * scale, f'band {bi}, rows {r0}..{r1}: gradient error {err:.3e} of {scale:.3e}'
        worst = max(worst, err / scale)
        grad[0, bi:bi + 1, s0:s1] = 0.0
    assert not bool(grad.any()), 'gradient outside the bands'
    lc += (count - band_count) * 0.01 ** 0.4 / max(count, 1)                # D = 0: every other masked pixel
    for k, v in ((0, lc), (1, ls), (3, lc / 2 + ls / 4)):
        assert sums[k] == pytest.approx(v, rel=1e-5), (k, sums[k], v)
    print(f'past 2^31: census element 2^31 in image {b31} row {y31}; loss {sums[3]:.9g} (oracle {lc / 2 + ls / 4:.9g}), '
          f'worst band gradient error {worst:.2e}; call {seconds * 1e3:.1f} ms, peak device memory {peak / GB:.2f} GB '
          f'({torch.cuda.get_device_name()})')
    del census, img, flows, grad, occ
    _release()
