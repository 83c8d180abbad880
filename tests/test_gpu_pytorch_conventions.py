"""RAFT(conventions='pytorch') on the GPU: the grid_sample lookup kernels against their NumPy float32 emulation (bit for
bit) and fp64 grid_sample, the encoders under PyTorch padding and epsilon against the PyTorch-layout fp64 oracle, the
whole model loaded from a synthetic `.pth` against that oracle, its plumbing, and the unchanged default."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cases
from oracle import raft_pytorch as rp

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope='module')
def T():
    import tf_raft_b200
    from tf_raft_b200 import _lib
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    return tf_raft_b200


@pytest.fixture(scope='module')
def ckpt():
    return rp.synthetic_checkpoint(seed=7)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).cuda()


# --------------------------------------------------------------------------------------------- 1. lookup kernels
def _pyramid(b, h, w, levels, seed):
    f1, f2 = cases.fmaps(b, h, w, 32, seed)
    pyr = rp.corr_pyramid(torch.from_numpy(f1).permute(0, 3, 1, 2).double(),
                          torch.from_numpy(f2).permute(0, 3, 1, 2).double(), levels)
    return [p[:, 0].float().numpy() for p in pyr]


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


def _lookup(T, pyr, coords, radius, sampler, fn='corr_lookup_ex'):
    from tf_raft_b200 import _lib
    b, h, w, _ = coords.shape
    levels = len(pyr)
    nch = levels * (2 * radius + 1) ** 2
    out = torch.full((b, h, w, nch), 7.0, device='cuda')
    dp = [dev(p) for p in pyr]
    args = [_lib.ptr_array(dp), _lib.ptr(dev(coords)), b, h, w, levels, radius, _lib.ptr(out), nch]
    if fn == 'corr_lookup_ex':
        args.append(sampler)
    _lib.call(fn, out.device, *args)
    torch.cuda.synchronize()
    return out.cpu().numpy()


LOOKUP_CASES = [(g, levels, r) for levels, grids in cases.LOOKUP_GRIDS.items() for g in grids
                for r in ((4, 3, 2) if levels == 4 else (4,))]


@pytest.mark.parametrize('grid,levels,radius', LOOKUP_CASES, ids=lambda v: 'x'.join(map(str, v)) if isinstance(v, tuple) else str(v))
@pytest.mark.parametrize('kind', ['grid', 'jitter', 'edge', 'special'])
def test_lookup_bit_exact_against_emulation_and_fp64(T, grid, levels, radius, kind):
    b, h, w = grid
    pyr = _pyramid(b, h, w, levels, seed=levels)
    if kind == 'special':                                 # NaN texels inside and just outside footprints
        pyr[0].reshape(-1)[::97] = np.nan
        pyr[-1].reshape(-1)[::13] = np.nan
    coords = _coords(b, h, w, kind)
    got = _lookup(T, pyr, coords, radius, 1)
    want = rp.lookup_emulated(pyr, coords, radius)
    path = cases.lookup_path(b, h, w, levels, radius, levels * (2 * radius + 1) ** 2)
    # bit for bit; a NaN is compared as a NaN (the device's canonical NaN has another payload than NumPy's)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=f'{path} kernel: NaN positions')
    np.testing.assert_array_equal(np.where(np.isnan(got), 0, got).view(np.uint32),
                                  np.where(np.isnan(want), 0, want).astype(F32).view(np.uint32), err_msg=f'{path} kernel')
    # fp64 grid_sample from the same fp32 coordinates: within a few ulps of sum |w v| plus the coordinates' own rounding
    if kind != 'special':
        t = torch.from_numpy(coords).double().permute(0, 3, 1, 2)
        p64 = [torch.from_numpy(p).double()[:, None] for p in pyr]
        ref = rp.corr_lookup(p64, t, radius).permute(0, 2, 3, 1).numpy()
        mag = rp.corr_lookup([p.abs() for p in p64], t, radius).permute(0, 2, 3, 1).numpy()
        vmax = max(float(np.abs(p).max()) for p in pyr)
        cmag = np.abs(np.nan_to_num(coords, posinf=0, neginf=0)).max(-1, keepdims=True) / 1.0
        bound = 8 * 2.0 ** -24 * (mag + (np.minimum(cmag, max(h, w)) + 2) * vmax)
        assert np.all(np.abs(got - ref) <= bound), float(np.abs(got - ref).max())


def test_normalisation_is_pytorchs_on_the_device(T):
    """The sampler's g is what RAFT's own expression `2 * xgrid / (W - 1) - 1` gives on CUDA float32 tensors (a Python
    int divisor), bit for bit: ATen divides by such a scalar as a product with its fp32 reciprocal."""
    rng = np.random.default_rng(12)
    v = np.concatenate([rng.uniform(-80, 80, 200000), rng.integers(-80, 80, 20000) + 0.5 * rng.integers(0, 2, 20000),
                        rng.uniform(-1e6, 1e6, 20000)]).astype(F32)
    for n in (2, 3, 7, 13, 31, 46, 62, 64, 100, 127):
        x = torch.from_numpy(v).cuda()
        got = (2 * x / (n - 1) - 1).cpu().numpy()
        with np.errstate(all='ignore'):
            want = (F32(2) * v) * (F32(1) / F32(n - 1)) - F32(1)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), n


def test_lookup_levels_of_size_one_are_zero(T):
    pyr = _pyramid(2, 9, 13, 4, seed=1)                      # levels 9x13, 4x6, 2x3, 1x1
    pyr2 = _pyramid(2, 9, 1, 1, seed=1)
    for p, coords, r in ((pyr, cases.lookup_coords(2, 9, 13, 'jitter'), 4), (pyr2, cases.lookup_coords(2, 9, 1, 'jitter'), 3)):
        got = _lookup(T, p, coords, r, 1)
        nt = (2 * r + 1) ** 2
        for l, lv in enumerate(p):
            if min(lv.shape[1:]) == 1:
                assert not got[..., l * nt:(l + 1) * nt].any()


def test_default_sampler_unchanged(T):
    for (b, h, w), levels, r in [((2, 9, 13), 4, 4), ((1, 8, 32), 4, 3), ((2, 7, 3), 2, 4)]:
        pyr = _pyramid(b, h, w, levels, seed=3)
        coords = cases.lookup_coords(b, h, w, 'edge')
        old = _lookup(T, pyr, coords, r, 0, fn='corr_lookup')
        new = _lookup(T, pyr, coords, r, 0)
        assert np.array_equal(old.view(np.uint32), new.view(np.uint32))


# --------------------------------------------------------------------------------------------- 2. encoders
# cases.ENCODER_GRIDS puts a stride-2 convolution on every (pixel tile, input-height parity, input-width parity) with
# its output two tiles or more each way, so every tile meets the odd, negative first tap coordinate of PyTorch's
# symmetric padding; the even sizes are where the two paddings differ on both axes from the stem on.
ENC_GRIDS = list(cases.ENCODER_GRIDS) + [(64, 64), (96, 128), (48, 80), (448, 512)]
_REF = {}


def _encoder_ref(ckpt, images, prefix, kind, key):
    """fp64 output, and the largest 1 / sqrt(var + eps) of the instance norms: the factor by which a norm amplifies an
    error in its input.  It is about 7 on these images, but 1 / sqrt(1e-5) = 316 where the last stage has two pixels
    (8x9, 9x8) and a channel holds two nearly equal values."""
    if key not in _REF:
        x = torch.from_numpy(images).double().permute(0, 3, 1, 2)
        x = 2 * (x / 255.0) - 1.0
        gain = [1.0]
        norm = rp._norm

        def measured(sd, y, name, k):
            if k == 'instance':
                gain[0] = max(gain[0], float(torch.rsqrt(y.var(dim=(2, 3), unbiased=False) + 1e-5).max()))
            return norm(sd, y, name, k)
        rp._norm = measured
        try:
            with torch.no_grad():
                out = rp.encoder(rp._sd(ckpt, torch.float64), x, prefix, kind).permute(0, 2, 3, 1).numpy()
        finally:
            rp._norm = norm
        _REF[key] = out, gain[0]
    return _REF[key]


@pytest.mark.parametrize('backend', ['native', 'torch'])
@pytest.mark.parametrize('norm', ['instance', 'batch'])
@pytest.mark.parametrize('HW', ENC_GRIDS, ids=lambda v: f'{v[0]}x{v[1]}')
def test_encoders_against_fp64(T, ckpt, backend, norm, HW):
    H, W = HW
    if norm == 'instance' and (H, W) == (8, 8):
        pytest.skip('a 1x1 last stage: nn.InstanceNorm2d itself refuses one pixel, so PyTorch RAFT has no value here')
    params = T.load_pytorch_checkpoint(ckpt)
    prefix = 'fnet' if norm == 'instance' else 'cnet'
    enc = T.BasicEncoder(output_dim=256, norm_type=norm, backend=backend, conventions='pytorch', device='cuda')
    enc.load_params(params, prefix + '.')
    im, _ = cases.images(2, H, W)
    got = enc(dev(im), training=False, raw_image=True)
    torch.cuda.synchronize()
    want, gain = _encoder_ref(ckpt, im, prefix, norm, (H, W, norm))
    err = float(np.abs(got.cpu().numpy() - want).max())
    scale = max(1.0, float(np.abs(want).max()))
    print(f'{backend} {norm} {H}x{W}: max-abs {err:.2e} (max |ref| {scale:.2f}, norm gain {gain:.1f})')
    # the gate of the tf-raft encoder tests at a norm gain up to 8, widened in proportion beyond it
    assert err <= 2e-4 * scale * max(1.0, gain / 8)
    if backend == 'native':                            # each image bit for bit independent of its batch
        one = enc(dev(im[1:]), training=False, raw_image=True)
        assert torch.equal(one[0], got[1])


def test_encoder_prepare_ex_default_unchanged(T, ckpt):
    from tf_raft_b200 import _lib
    im, _ = cases.images(2, 64, 96)
    enc = T.BasicEncoder(output_dim=256, norm_type='batch', device='cuda', seed=5)
    new = enc(dev(im), training=False, raw_image=True)
    w = enc.prepared()
    old_blob = torch.empty_like(w)
    enc._prepared = None
    enc.prepared()                                     # rebuild through prepare_ex(TF), identical bytes
    assert torch.equal(enc._prepared, w)
    # the old entry point into another buffer
    import ctypes
    wts = _lib.RaftEncoderWeights()
    wts.conv1 = enc._conv_struct('conv1'); wts.norm1 = enc._norm_struct('norm1')
    k = 0
    for li, (_, stride) in enumerate(enc._stages, start=1):
        for bi, st in enumerate((stride, 1)):
            p = f'layer{li}.{bi}'
            blk = wts.block[k]
            blk.conv1, blk.conv2 = enc._conv_struct(p + '.conv1'), enc._conv_struct(p + '.conv2')
            blk.norm1, blk.norm2 = enc._norm_struct(p + '.norm1'), enc._norm_struct(p + '.norm2')
            if st != 1:
                blk.downsample = enc._conv_struct(p + '.downsample.0')
                blk.downsample_norm = enc._norm_struct(p + '.downsample.1')
            k += 1
    wts.conv2 = enc._conv_struct('conv2')
    _lib.call('encoder_prepare', old_blob.device, enc._variant, 2, 256, ctypes.cast(ctypes.pointer(wts), ctypes.c_void_p),
              _lib.ptr(old_blob), old_blob.numel())
    torch.cuda.synchronize()
    assert torch.equal(old_blob, w)
    enc._prepared = old_blob
    again = enc(dev(im), training=False, raw_image=True)
    assert torch.equal(again, new)


# --------------------------------------------------------------------------------------------- 3. the model
def _model(T, ckpt, tmp_path, precision, **kw):
    path = tmp_path / 'raft-synthetic.pth'
    torch.save(ckpt, path)
    m = T.RAFT(conventions='pytorch', precision=precision, device='cuda', **kw)
    m.load_pytorch_weights(str(path))
    return m


E2E = [
    ('448x512-b4-f16x2', 4, 448, 512, 12, 'f16x2', False),
    ('448x512-b4-fp32', 4, 448, 512, 12, 'fp32', False),
    ('64x64', 1, 64, 64, 12, 'f16x2', False),
    ('440x1024-warm', 1, 440, 1024, 12, 'f16x2', True),
]


@pytest.mark.parametrize('name,b,H,W,iters,precision,warm', E2E, ids=[e[0] for e in E2E])
def test_end_to_end_against_fp64(T, ckpt, tmp_path, name, b, H, W, iters, precision, warm):
    im1, _ = cases.images(b, H, W)
    im2 = np.roll(im1, (3, -5), axis=(1, 2)).copy()
    flow_init = None
    if warm:
        flow_init = np.random.default_rng(9).uniform(-2, 2, (b, H // 8, W // 8, 2)).astype(F32)
    m = _model(T, ckpt, tmp_path, precision, iters_pred=iters)
    got = m([dev(im1), dev(im2)], training=False, last_only=True,
            flow_init=None if flow_init is None else dev(flow_init))[-1]
    torch.cuda.synchronize()
    want = rp.forward(ckpt, im1, im2, iters, flow_init)[0][-1]
    err = np.abs(got.cpu().numpy() - want)
    print(f'{name}: worst final-flow error vs fp64 {err.max():.3e} (|flow| max {np.abs(want).max():.2f})')
    assert err.max() <= 1e-3


def test_plumbing_bit_for_bit(T, ckpt, tmp_path):
    im1, im2 = cases.images(2, 64, 96)
    m = _model(T, ckpt, tmp_path, 'f16x2', iters_pred=4)
    a, b = dev(im1), dev(im2)
    full = [f.clone() for f in m([a, b], training=False)]
    last = m([a, b], training=False, last_only=True)[-1].clone()
    assert torch.equal(last, full[-1])
    g = _model(T, ckpt, tmp_path, 'f16x2', iters_pred=4, use_graph=True)
    for _ in range(2):
        assert torch.equal(g([a, b], training=False, last_only=True)[-1], full[-1])
    fw, bw, _, _ = m.predict_bidirectional([a, b])
    assert torch.equal(fw, full[-1])
    assert torch.equal(bw, m([b, a], training=False, last_only=True)[-1])
    frames = [dev(x) for x in (im1, im2, np.roll(im2, 2, axis=2).copy())]
    video = [f.clone() for f in m.predict_video(frames, warm_start=False)]
    for t in range(2):
        assert torch.equal(video[t], m([frames[t], frames[t + 1]], training=False, last_only=True)[-1])


@pytest.mark.parametrize('precision', ['f16x2', 'fp32'])
@pytest.mark.parametrize('grid', [(9, 128), (13, 11)], ids=lambda g: f'{g[0]}x{g[1]}')
def test_fused_loop_equals_the_public_ops(T, ckpt, tmp_path, grid, precision):
    """raft_b200_forward_loop_ex(..., RAFT_SAMPLER_GRID) -- the grid window lookup writing fp16 hi/lo operands with the
    convf1 im2col rider on f16x2, fused coords1 += delta, mask head skipped where no prediction is asked for -- gives,
    byte for byte, what the loop spelled out with CorrBlock(sampler='grid_sample').retrieve, update_block and
    upsample_flow gives, at every iteration and with last_only=True."""
    h, w = grid
    iters, bs = 3, 2
    im1, im2 = cases.images(bs, 8 * h, 8 * w, 3, 4)
    a, b = dev(im1), dev(im2)
    model = _model(T, ckpt, tmp_path, precision, iters=iters, iters_pred=iters)
    fmap1, fmap2, net, inp = model._encode(a, b, False)
    cb = T.CorrBlock(fmap1, fmap2, model.corr_levels, model.corr_radius, precision=precision, sampler='grid_sample')
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
        assert torch.equal(full[i], ups[i]), f'iteration {i}: max-abs {float((full[i] - ups[i]).abs().max()):.3e}'
    last = model([a, b], training=False, last_only=True)
    assert len(last) == 1 and torch.equal(last[0], ups[-1]), 'last_only differs from the loop spelled out'


def test_forward_loop_ex_default_unchanged(T, tmp_path):
    from tf_raft_b200 import _lib
    im1, im2 = cases.images(1, 64, 96)
    m = T.RAFT(precision='f16x2', device='cuda', iters_pred=3, seed=4)
    new = m([dev(im1), dev(im2)], training=False)[-1].clone()
    old_loop = m._loop

    def loop(corr_block, net, inp, coords1, flow_ups, b, h, w):
        ub = m.update_block
        ws = ub.workspace(b, h, w)
        _lib.call('forward_loop', net.device, m._variant, _lib.ptr(ub.prepared()), _lib.ptr_array(corr_block.corr_pyramid),
                  m.corr_levels, m.corr_radius, _lib.ptr(net), _lib.ptr(inp), _lib.ptr(coords1), _lib.ptr_array(flow_ups),
                  len(flow_ups), b, h, w, _lib.ptr(ws), ws.numel(), m.precision)
    m._loop = loop
    old = m([dev(im1), dev(im2)], training=False)[-1]
    m._loop = old_loop
    assert torch.equal(old, new)


def test_conventions_guards(T, ckpt, tmp_path):
    with pytest.raises(ValueError, match='bottleneck'):
        T.SmallRAFT(conventions='pytorch', device='cuda')
    with pytest.raises(ValueError):
        T.RAFT(conventions='keras', device='cuda')
    path = tmp_path / 'r.pth'
    torch.save(ckpt, path)
    with pytest.raises(ValueError, match="conventions='pytorch'"):
        T.RAFT(device='cuda').load_pytorch_weights(str(path))
    m = _model(T, ckpt, tmp_path, 'f16x2')
    with pytest.raises(NotImplementedError):
        m.compile(optimizer=None)
    with pytest.raises(NotImplementedError):
        m.train_step(None)
