"""Non-finite and out-of-range operands, against the oracle in float64.

Every other GPU test draws its operands from one narrow band (N(0, 1) features, tanh / relu / 3-sigma update inputs,
Glorot weights).  Here:

* NaN is a data-flow tracer.  The set of outputs one planted NaN reaches is the receptive field of that input through
  every convolution's zero padding, the TMA zero fill, the stride-2 asymmetric padding, the pixel-tile halos of the
  update mega-kernel and the 128-query tiles of the correlation kernel, and it must never cross into another image.  The
  kernels' NaN masks must equal the fp64 oracle's exactly (tests/test_value_cases.py shows that the oracle's masks are
  the receptive fields), so these checks need no tolerance.  They also pin the NaN contract of DESIGN section 4: the
  fp16 hi/lo split and every ReLU keep NaN.
* A magnitude sweep checks that the tensor-core kernels follow their own split arithmetic (cases.split_f16) at every
  scale, subnormal fp16 hi / lo and saturation at 65504 included, and measures where the product stays fp32-grade.
* Scaling a last layer's weights and bias by 2^s must scale its output by exactly 2^s: the packing's per-layer 2^k
  absorbs it.
"""
import os
import subprocess

import numpy as np
import pytest
import torch

import cases
import probe_build
from oracle import raft_torch as rt, weights
from test_gpu_geometry import PRECISIONS, UPDATE_TOL, _grid_id, dev, lookup_forward_matrix, maxabs, nchw, nhwc

pytestmark = pytest.mark.gpu
F64 = torch.float64
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
PROBE_SRC = os.path.join(ROOT, 'tests', 'values_probe.cu')


@pytest.fixture(scope='module')
def T():
    import tf_raft_b200
    from tf_raft_b200 import _lib
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    return tf_raft_b200


def same(a, b):
    """Equal values with NaN equal to NaN (NaN payloads may differ)."""
    a, b = a.detach().cpu(), b.detach().cpu()
    na, nb = torch.isnan(a), torch.isnan(b)
    return a.shape == b.shape and torch.equal(na, nb) and torch.equal(a[~na], b[~nb])


# ------------------------------------------------------------------------------------------ 1. ReLU and split, bit for bit
@pytest.fixture(scope='module')
def probe():
    exe = probe_build.build(PROBE_SRC, 'raft_values_probe')
    assert exe is not None, 'nvcc not found'
    return exe


def _specials():
    f = np.float32
    vals = [0.0, -0.0, 1.0, -1.0, 2.0 ** -126, -(2.0 ** -126), 2.0 ** -149, -(2.0 ** -149), 3.4e38, -3.4e38,
            np.inf, -np.inf, 65504.0, -65504.0, 65519.99, 65520.0, 1e5, -1e5, 2.0 ** -14, 2.0 ** -24, 2.0 ** -25,
            3 * 2.0 ** -26, 1 + 2.0 ** -20, 1 / 3, -7.25]
    bits = [int(np.array(v, dtype=f).view(np.uint32)) for v in vals]
    bits += [0x7fc00000, 0xffc00000, 0x7f800001, 0x7fbfffff, 0xff812345]          # quiet / signalling, both signs
    bits += np.random.default_rng(0).integers(0, 2 ** 32, 64, dtype=np.uint64).astype(int).tolist()
    return bits


def test_relu_and_split_special_values(probe):
    """relu_nan gives NaN for NaN and fmaxf(v, 0)'s exact bits for every other input (-0 -> +0, subnormals, inf).  The
    split gives NaN for NaN and otherwise the NumPy emulation's exact bits (saturation at +-65504 of everything beyond,
    inf included); split_f16x2 gives split_f16's bits in both lanes."""
    bits = _specials()
    res = subprocess.run([probe] + ['%08x' % b for b in bits], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0, res.stderr
    rows = [[int(t, 16) for t in line.split()] for line in res.stdout.splitlines()]
    assert len(rows) == len(bits)
    for b, (relu, fmax, hi, lo, h0, l0, h1, l1) in zip(bits, rows):
        v = np.array(b, dtype=np.uint32).view(np.float32)
        f16 = lambda x: np.array(x, dtype=np.uint16).view(np.float16)
        if np.isnan(v):
            assert np.isnan(np.array(relu, dtype=np.uint32).view(np.float32)), hex(b)
            assert np.isnan(f16(hi)) and np.isnan(f16(h0)) and np.isnan(f16(h1)), hex(b)
            continue
        assert relu == fmax, (hex(b), hex(relu), hex(fmax))
        assert (h0, l0) == (hi, lo), hex(b)
        for (gh, gl), x in (((hi, lo), v), ((h1, l1), -v)):
            eh, el = cases.split_f16(np.array([x], dtype=np.float32))
            assert (gh, gl) == (int(eh.view(np.uint16)[0]), int(el.view(np.uint16)[0])), (hex(b), float(x))


# ------------------------------------------------------------------------------------------ 2. correlation pyramid
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('case', [cases.PYRAMID_CASES[2], cases.PYRAMID_CASES[3], cases.PYRAMID_CASES[4]],
                         ids=_grid_id)
def test_pyramid_nan_tracer(T, case, precision):
    """A NaN in fmap1[1, q] (last channel, a query in the last, ragged 128-query tile of image 1) and one in fmap2[0, n]
    (last channel): every level's NaN mask equals the fp64 oracle's -- row q everywhere, the column of n in image 0
    only, pooled into the cells that contain it -- and the finite values keep the 2e-5 of test_gpu_geometry.  The
    correlation kernel tiles the queries of each image separately (mtiles_img, corr_tc.cuh), so no tile straddles two
    images; the ragged last tile, whose rows past the image are TMA zero fill, is where a stray row would show."""
    b, h, w, c, levels = case
    N = h * w
    f1, f2 = cases.fmaps(b, h, w, c, seed=10 + c + levels)
    q = min(N - 1, (N // 128) * 128 + 5)                     # inside image 1's last query tile
    f1[1].reshape(N, c)[q, c - 1] = np.nan
    f2[0].reshape(N, c)[N - w - 2, c - 1] = np.nan           # a cell in the last-but-one row, beside the ragged edge
    cb = T.CorrBlock(dev(f1), dev(f2), num_levels=levels, radius=4, precision=precision)
    truth = rt.CorrBlock(torch.from_numpy(f1).double(), torch.from_numpy(f2).double(), levels, 4).corr_pyramid
    for l in range(levels):
        got, want = cb.corr_pyramid[l].cpu(), truth[l]
        nan = torch.isnan(want)
        assert nan[N + q].all() and not nan[2 * N:].any()
        assert torch.equal(torch.isnan(got), nan), f'level {l}: {int((torch.isnan(got) != nan).sum())} NaN positions differ'
        np.testing.assert_allclose(got[~nan].numpy(), want[~nan].numpy(), atol=2e-5, rtol=2e-5, err_msg=f'level {l}')


# ------------------------------------------------------------------------------------------ 3. lookup
def _plant_non_finite(pyr):
    rng = np.random.default_rng(len(pyr))
    for p in pyr:
        flat = p.reshape(-1)
        idx = rng.choice(flat.size, size=min(flat.size, 6), replace=False)
        flat[idx[:3]] = np.nan
        flat[idx[3:]] = np.inf


def test_lookup_nan_and_inf_bit_exact(T):
    """The bit-exact lookup matrix of test_gpu_geometry on a pyramid with NaN and +inf cells: the reference expression's
    0 * v taps carry them into zero-weight taps too, and the kernels must land NaN / inf on exactly the same outputs."""
    from test_gpu_geometry import KINDS, RADII
    n = lookup_forward_matrix(T, plant=_plant_non_finite)
    assert n == len(RADII) * len(KINDS) * sum(len(g) for g in cases.LOOKUP_GRIDS.values())


# ------------------------------------------------------------------------------------------ 4. update blocks per tile
INPUTS = ('net', 'inp', 'corr', 'flow')


@pytest.fixture(scope='module')
def update_cache():
    cache = {}

    def get(key, make):
        if key not in cache:
            cache[key] = make()
        return cache[key]
    return get


@pytest.mark.parametrize('which', INPUTS)
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('form', ['basic', 'basic-no-mask', 'small'])
@pytest.mark.parametrize('grid', cases.TILE_GRIDS, ids=_grid_id)
def test_update_block_nan_tracer(T, update_cache, grid, form, precision, which):
    """One NaN in one input, in image 1, in the last real channel, at the bottom-right pixel of the first pixel tile (so
    its halo crosses into the neighbouring tiles): net / mask / delta NaN masks equal the fp64 oracle's, the finite
    values keep UPDATE_TOL, and the other images are bit-identical to a run without the NaN."""
    variant = 'small' if form == 'small' else 'raft'
    b, h, w = grid
    tw, th = cases.tc_tile(h, w)
    y, x = min(th, h) - 1, min(tw, w) - 1
    p = update_cache(('params', variant), lambda: weights.init_params(variant, 1234, bias_scale=0.05))
    clean = cases.update_inputs(variant, b, h, w, seed=20 + h * w)
    k = INPUTS.index(which)
    ins = [a.copy() for a in clean]
    ins[k][1, y, x, -1] = np.nan

    def oracle():
        fn = rt.basic_update_block if variant == 'raft' else rt.small_update_block
        net, mask, delta = fn(rt.Ops(p, F64), *[nchw(a, F64) for a in ins])
        return dict(net=nhwc(net), mask=nhwc(mask), delta=nhwc(delta))
    truth = update_cache((variant, grid, which), oracle)

    def block():
        blk = (T.BasicUpdateBlock if variant == 'raft' else T.SmallUpdateBlock)(precision=precision)
        blk.load_params(p, 'update_block.')
        return blk
    blk = update_cache((form, precision), block)

    def run(arrays):
        args = [dev(a) for a in arrays]
        out = blk(args, compute_mask=form == 'basic') if variant == 'raft' else blk(args)
        return dict(zip(('net', 'mask', 'delta'), (None if t is None else t.cpu() for t in out)))
    got, ref = run(ins), run(clean)
    others = [i for i in range(b) if i != 1]
    for key, g in got.items():
        if g is None:
            continue
        want = truth[key]
        nan = torch.isnan(want)
        assert nan[1].any() and not nan[others].any(), key
        assert torch.equal(torch.isnan(g), nan), \
            f'{key}: {int((torch.isnan(g) != nan).sum())} NaN positions differ from the oracle (tile {tw}x{th})'
        e = maxabs(g[~nan], want[~nan])
        assert e < UPDATE_TOL[key], (key, e)
        assert torch.equal(g[others], ref[key][others]), f'{key}: another image of the batch changed'


# ------------------------------------------------------------------------------------------ 5. encoders
@pytest.mark.parametrize('size', [(70, 98), (36, 52)], ids=_grid_id)
@pytest.mark.parametrize('norm', [None, 'batch-inference', 'instance', 'batch-training'])
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_encoder_nan_tracer(T, variant, norm, size):
    """One NaN pixel in image 1 of 3 (raw 0..255 input, odd stride-2 sizes).  No norm and inference BatchNorm (folded
    into the epilogue): exactly the oracle's NaN mask, the rest within the 2e-4 of test_gpu_geometry.  Instance norm:
    image 1 is all NaN, the others bit-identical to a clean run.  Training BatchNorm: the whole batch is NaN."""
    from tf_raft_b200.layers.extractor import BasicEncoder, SmallEncoder
    H, W = size
    out_dim = 256 if variant == 'raft' else 128
    nt = norm.split('-')[0] if norm else None
    training = norm == 'batch-training'
    p = cases.encoder_params(variant, nt, out_dim, seed=99 + H)
    clean, _ = cases.images(3, H, W, seed0=H + W)
    im = clean.copy()
    im[1, H // 2 + 1, W - 1, 2] = np.nan
    enc = (BasicEncoder if variant == 'raft' else SmallEncoder)(output_dim=out_dim, norm_type=nt, backend='native')
    enc.load_params(p, 'enc.')
    got = enc(dev(im), training=training, raw_image=True).cpu()
    ref = enc(dev(clean), training=training, raw_image=True).cpu()
    nan = torch.isnan(got)
    if norm == 'batch-training':
        assert nan.all()
        return
    if norm == 'instance':
        assert nan[1].all() and not nan[[0, 2]].any() and torch.equal(got[[0, 2]], ref[[0, 2]])
        return
    x = (2 * (torch.from_numpy(im).double() / 255.0) - 1.0).permute(0, 3, 1, 2)
    truth = nhwc(rt.encoder(rt.Ops(p, F64), x, 'enc', nt, False))
    want = torch.isnan(truth)
    assert want[1].any() and not want[[0, 2]].any()
    assert torch.equal(nan, want), f'{int((nan != want).sum())} NaN positions differ from the oracle'
    assert maxabs(got[~want], truth[~want]) < 2e-4
    assert torch.equal(got[[0, 2]], ref[[0, 2]])


def test_context_split_keeps_nan(T):
    """net = tanh, inp = relu of the context encoder output (model.py:84-86): NaN stays NaN in both, -0 -> +0 in inp."""
    from tf_raft_b200 import _lib
    hid, ctx, n = 96, 64, 37
    c = torch.randn(n, hid + ctx, generator=torch.Generator().manual_seed(0))
    c[3, 5] = c[4, hid + 7] = float('nan')
    c[5, hid + 1] = -0.0
    c[6, hid + 2], c[7, hid + 3] = float('inf'), float('-inf')
    cd = dev(c)
    net = torch.empty((n, hid), device='cuda')
    inp = torch.empty((n, ctx), device='cuda')
    _lib.check(_lib.lib().raft_b200_context_split(_lib.ptr(cd), n, hid, ctx, _lib.ptr(net), _lib.ptr(inp),
                                                  _lib.stream()), 'context_split')
    net, inp = net.cpu(), inp.cpu()
    assert torch.equal(torch.isnan(net), torch.isnan(c[:, :hid])) and torch.equal(torch.isnan(inp), torch.isnan(c[:, hid:]))
    want = c[:, hid:].clamp_min(0)
    assert same(inp, want) and not torch.signbit(inp[~torch.isnan(inp)]).any()
    assert maxabs(net[~torch.isnan(net)], torch.tanh(c[:, :hid])[~torch.isnan(net)]) < 1e-6


# ------------------------------------------------------------------------------------------ 6. fused loop
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_fused_loop_nan_equals_the_public_ops(T, monkeypatch, variant, precision):
    """test_gpu_geometry's fused-loop identity with non-finite values planted three ways: a NaN in one fmap1 element
    of image 1; NaN and +inf cells in image 1's rows of every pyramid level (the fused loop's lookup writes them as the
    fp16 hi/lo operands of convc1, the spelled-out loop as fp32 values that the update block splits); and, for RAFT, a
    NaN weight of mask logit 100 in mask.2 (through the weight packing), which makes that logit NaN at every pixel of
    both images.  The fused loop and the loop spelled out with the public ops give the same NaN masks and the same finite
    values at every iteration and with last_only.  Image 0 is NaN exactly where the NaN logit reaches -- sub-pixel
    (1, 3) of every 8 x 8 block for RAFT, nowhere for SmallRAFT -- so the planted feature and pyramid cells of image 1
    never reach it."""
    from tf_raft_b200 import model as model_module
    h, w = 13, 11
    iters, bs = 3, 2
    p = weights.init_params(variant, 1234, bias_scale=0.05, norm_jitter=0.1)
    if variant == 'raft':
        p['update_block.mask.2.kernel'] = p['update_block.mask.2.kernel'].copy()
        p['update_block.mask.2.kernel'][0, 0, 17, 100] = np.nan
    im1, im2 = cases.images(bs, 8 * h, 8 * w, 3, 4)
    a, b = dev(im1), dev(im2)
    model = (T.RAFT if variant == 'raft' else T.SmallRAFT)(iters=iters, iters_pred=iters, precision=precision)
    model.load_params(p)
    encode = model._encode

    def planted(i1, i2, training):
        f1, f2, net, inp = encode(i1, i2, training)
        f1[1, 4, 6, 3] = float('nan')
        return f1, f2, net, inp
    model._encode = planted
    n = h * w

    class PlantedCorrBlock(T.CorrBlock):
        def __init__(self, *args, **kw):
            super().__init__(*args, **kw)
            for l, pyr in enumerate(self.corr_pyramid):
                pyr[n + 3 + l, 0, 0, 0] = float('inf')
                pyr[n + 17, -1, -1, 0] = float('nan')
                pyr[2 * n - 1, pyr.shape[1] // 2, pyr.shape[2] // 2, 0] = float('inf')
    monkeypatch.setattr(model_module, 'CorrBlock', PlantedCorrBlock)
    fmap1, fmap2, net, inp = model._encode(a, b, False)
    cb = PlantedCorrBlock(fmap1, fmap2, model.corr_levels, model.corr_radius, precision=precision)
    coords1 = T.coords_grid(bs, h, w)
    grid0 = coords1.clone()
    ups = []
    for _ in range(iters):
        corr = cb.retrieve(coords1)
        net, mask, delta = model.update_block([net, inp, corr, coords1 - grid0])
        coords1 = coords1 + delta
        ups.append(model.upsample_flow(coords1 - grid0, mask))
    # image 0: for RAFT the NaN logit (channel 100 = sub-pixel (1, 3), tap 1) reaches that sub-pixel of every 8 x 8 block
    img0 = torch.zeros((8 * h, 8 * w, 2), dtype=torch.bool)
    if variant == 'raft':
        img0[1::8, 3::8] = True
    full = model([a, b], training=False)
    for i in range(iters):
        assert torch.isnan(ups[i][1]).any() and torch.equal(torch.isnan(ups[i][0]).cpu(), img0), i
        assert same(full[i], ups[i]), f'iteration {i}'
    last = model([a, b], training=False, last_only=True)
    assert len(last) == 1 and same(last[0], ups[-1])


# ------------------------------------------------------------------------------------------ 7. magnitude sweep
SCALES = (-16, -10, -6, -3, 0, 4, 7)
FP32_GRADE = (-6, -3, 0, 4, 7)          # the scales where the f16x2 pyramid keeps the fp32-grade 2e-5 (scaled by 2^2s)


def _pool(f):
    """2 x 2 VALID average pooling of (h, w, C) features in fp32, in the order of corr_prep_kernel: ((a + b) + (c + d))
    * 0.25 with a, b the upper row."""
    h, w = f.shape[0] // 2 * 2, f.shape[1] // 2 * 2
    f = f[:h, :w]
    return (((f[0::2, 0::2] + f[0::2, 1::2]) + (f[1::2, 0::2] + f[1::2, 1::2])) * np.float32(0.25)).astype(np.float32)


@pytest.mark.parametrize('scale', SCALES + ('1e5',))
def test_pyramid_magnitude_sweep(T, scale):
    """Feature maps scaled by 2^s (and, for '1e5', N(0, 1) maps with +-1e5 planted: saturated at 65504): every level of
    the f16x2 pyramid equals the fp64 emulation of the split arithmetic to fp32 accumulation, 64 * 2^-24 * sum |a||b|
    / sqrt(C).  Against the fp64 truth the error scaled by 2^-2s keeps 2e-5 on FP32_GRADE and is printed for all."""
    b, h, w, c, levels = cases.PYRAMID_CASES[3]
    f1, f2 = cases.fmaps(b, h, w, c, seed=77)
    s = 0 if scale == '1e5' else scale
    f1, f2 = f1 * np.float32(2.0 ** s), f2 * np.float32(2.0 ** s)
    if scale == '1e5':
        f1[0, 3, 4, 10], f1[1, 0, 0, 0], f2[0, 5, 5, 10], f2[2, 7, 1, 200] = 1e5, -1e5, 1e5, -1e5
    cb = T.CorrBlock(dev(f1), dev(f2), num_levels=levels, radius=4, precision='f16x2')
    truth = rt.CorrBlock(torch.from_numpy(f1).double(), torch.from_numpy(f2).double(), levels, 4).corr_pyramid
    N = h * w
    worst, truth_err = 0.0, 0.0
    for i in range(b):
        a, g = f1[i].reshape(N, c), f2[i]
        for l in range(levels):
            if l:
                g = _pool(g)
            emu, mag = cases.split_product(a, g.reshape(-1, c))
            got = cb.corr_pyramid[l][i * N:(i + 1) * N].reshape(N, -1).cpu().numpy().astype(np.float64)
            dev_ = np.abs(got - emu / np.sqrt(c))
            tol = 64 * 2.0 ** -24 * mag / np.sqrt(c)
            worst = max(worst, float((dev_ / np.maximum(tol, 1e-300)).max()))
            assert (dev_ <= tol).all(), f'image {i} level {l}: {int((dev_ > tol).sum())} values off the split arithmetic'
            t = truth[l][i * N:(i + 1) * N].reshape(N, -1).numpy()
            truth_err = max(truth_err, float(np.abs(got - t).max()) / 2.0 ** (2 * s))
    print(f'scale {scale}: worst |pyramid - split emulation| / tolerance {worst:.3f}; '
          f'|pyramid - fp64| / 2^2s {truth_err:.2e}')
    if scale in FP32_GRADE:
        assert truth_err < 2e-5


LAST_LAYER_SCALES = (-7, 1, 9, 16)      # k of these layers is 16 or 17 unscaled: k - s stays inside the +-24 clamp


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('s', LAST_LAYER_SCALES)
def test_last_layer_weight_scale_is_exact(T, s, precision):
    """Weights and bias of flow_head.conv2 and mask.2 times 2^s scale delta and mask by exactly 2^s: each is a packed
    layer of its own, whose 2^k absorbs the factor (while k stays within its +-24 clamp), and the fp32 path scales every
    product exactly."""
    b, h, w = cases.TILE_GRIDS[3]
    p = weights.init_params('raft', 1234, bias_scale=0.05)
    q = dict(p)
    for name in ('update_block.flow_head.conv2', 'update_block.mask.2'):
        for part in ('kernel', 'bias'):
            q[f'{name}.{part}'] = (p[f'{name}.{part}'] * np.float32(2.0 ** s)).astype(np.float32)
    args = [dev(a) for a in cases.update_inputs('raft', b, h, w, seed=5)]
    outs = []
    for params in (p, q):
        blk = T.BasicUpdateBlock(precision=precision)
        blk.load_params(params, 'update_block.')
        outs.append(blk(args, compute_mask=True))
    (n0, m0, d0), (n1, m1, d1) = outs
    assert torch.equal(n0, n1)
    assert torch.equal(d1, d0 * 2.0 ** s) and torch.equal(m1, m0 * 2.0 ** s)


@pytest.mark.parametrize('s', LAST_LAYER_SCALES)
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_encoder_output_layer_weight_scale_is_exact(T, variant, s):
    """The encoder's 1x1 output convolution (conv2, a packed layer of its own): its weights and bias times 2^s scale
    the feature map by exactly 2^s."""
    from tf_raft_b200.layers.extractor import BasicEncoder, SmallEncoder
    out_dim = 256 if variant == 'raft' else 128
    p = cases.encoder_params(variant, 'instance', out_dim, seed=7)
    q = dict(p)
    for part in ('kernel', 'bias'):
        q[f'enc.conv2.{part}'] = (p[f'enc.conv2.{part}'] * np.float32(2.0 ** s)).astype(np.float32)
    im, _ = cases.images(2, 36, 52, seed0=3)
    outs = []
    for params in (p, q):
        enc = (BasicEncoder if variant == 'raft' else SmallEncoder)(output_dim=out_dim, norm_type='instance',
                                                                     backend='native')
        enc.load_params(params, 'enc.')
        outs.append(enc(dev(im), training=False, raw_image=True))
    assert torch.equal(outs[1], outs[0] * 2.0 ** s)


# Merged packed layers share one 2^k, set by the largest weight of all their parts (weight_scale_kernel): a part whose
# weights are 2^8 smaller than its partner's sits 2^8 below the [2^12, 2^13) window of the packing, and its lo residuals
# move 8 binades towards the fp16 subnormals.
MERGED = {
    'fh1|m0': ('update_block.mask.0', 8),         # the mask head 2^8 larger: fh1 (delta's path) is the small part
    'z|r1': ('update_block.gru.convz1', -8),       # convz1 2^8 smaller than convr1 in the first GRU pass
}


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('merged', sorted(MERGED))
def test_merged_layer_parts_of_different_magnitude(T, merged, precision):
    """One part of a merged packed layer scaled by 2^+-8 against its partner (weights only; the biases are applied in
    fp32 after the product): net, delta and mask stay within UPDATE_TOL of the fp64 oracle run with the same weights
    (the mask's tolerance scaled with the mask).  The errors are printed beside the fp32 oracle's."""
    name, s = MERGED[merged]
    b, h, w = cases.TILE_GRIDS[3]
    p = dict(weights.init_params('raft', 1234, bias_scale=0.05))
    p[name + '.kernel'] = (p[name + '.kernel'] * np.float32(2.0 ** s)).astype(np.float32)
    ins = cases.update_inputs('raft', b, h, w, seed=20 + h * w)
    truth, fp32 = [dict(zip(('net', 'mask', 'delta'), map(nhwc, rt.basic_update_block(rt.Ops(p, dt), *[nchw(a, dt) for a in ins]))))
                   for dt in (F64, torch.float32)]
    blk = T.BasicUpdateBlock(precision=precision)
    blk.load_params(p, 'update_block.')
    got = dict(zip(('net', 'mask', 'delta'), blk([dev(a) for a in ins], compute_mask=True)))
    scale = max(1.0, float(truth['mask'].abs().max()) / 0.5)
    errs = {k: (maxabs(got[k], truth[k]), maxabs(fp32[k], truth[k])) for k in got}
    print(f'{merged} 2^{s} {precision}: ' + ', '.join(f'{k} {e:.2e} (fp32 oracle {o:.2e})' for k, (e, o) in errs.items()))
    for k, (e, _) in errs.items():
        assert e < UPDATE_TOL[k] * (scale if k == 'mask' else 1.0), (k, errs)


class SplitOps(rt.Ops):
    """oracle.raft_torch.Ops with every convolution's activation operand split as the tensor-core path splits it
    (split_f16: saturate to +-65504, hi = fp16, lo = fp16 of the residual) and the weights exact: after their 2^k the
    packed weights sit in fp16's normal range, so their split is fp32-grade and is not what this emulation is for."""

    def __init__(self, params, dtype):
        f16 = lambda x: x.to(torch.float16).to(x.dtype)
        super().__init__(params, dtype, split=(f16, f16, lambda w: w, torch.zeros_like))

    def conv(self, x, name, stride=1, padding='same'):
        return super().conv(x.clamp(-65504, 65504), name, stride, padding)


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_corr_beyond_fp16_range(T, variant, precision):
    """corr times 2^13: about 0.8 % of its entries pass 65504, and the activations behind convc1 pass it too.  The fp32
    path matches the fp64 oracle.  The f16x2 path matches the fp64 oracle with every convolution's activation operand
    split and saturated as the kernels do (SplitOps) -- saturation at +-65504 is the documented behaviour, not an
    accident -- and is far from the unsaturated oracle.  This input is badly conditioned (pre-activations of order 1e5),
    so the bound is the larger of UPDATE_TOL and 4x the error of the same computation in fp32 against fp64."""
    b, h, w = cases.TILE_GRIDS[3]
    p = weights.init_params(variant, 1234, bias_scale=0.05)
    net, inp, corr, flow = cases.update_inputs(variant, b, h, w, seed=5)
    corr = (corr * np.float32(2.0 ** 13)).astype(np.float32)
    assert (np.abs(corr) > 65504).mean() > 0.005
    fn = rt.basic_update_block if variant == 'raft' else rt.small_update_block

    def oracle(dt, ops):
        outs = fn(ops(p, dt), *[nchw(a, dt) for a in (net, inp, corr, flow)])
        return dict(zip(('net', 'mask', 'delta'), map(nhwc, outs)))
    ops, other_ops = (rt.Ops, SplitOps) if precision == 'fp32' else (SplitOps, rt.Ops)
    want, want32, other = oracle(F64, ops), oracle(torch.float32, ops), oracle(F64, other_ops)
    blk = (T.BasicUpdateBlock if variant == 'raft' else T.SmallUpdateBlock)(precision=precision)
    blk.load_params(p, 'update_block.')
    args = [dev(a) for a in (net, inp, corr, flow)]
    out = blk(args, compute_mask=True) if variant == 'raft' else blk(args)
    got = {k: v for k, v in zip(('net', 'mask', 'delta'), out) if v is not None}
    for k in got:
        e, o, far = maxabs(got[k], want[k]), maxabs(want32[k], want[k]), maxabs(got[k], other[k])
        print(f'{variant} {precision} {k}: {e:.2e} (fp32 oracle {o:.2e}); against the other oracle {far:.2e}')
        assert e < max(UPDATE_TOL[k], 4 * o), (k, e, o)
    assert maxabs(got['net'], other['net']) > 0.1
