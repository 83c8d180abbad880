"""The original PyTorch RAFT-small on the GPU (SmallRAFT(conventions='pytorch', blocks='bottleneck')): the align-corners
upflow8 kernel against its NumPy float32 emulation (bit for bit), the bottleneck encoders on both backends against the
fp64 oracle, the whole model loaded from a synthetic raft-small.pth against `forward_small`, the fused loop against the
loop spelled out, its plumbing, its guards and RAFT's evaluation script."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cases
from oracle import raft_pytorch as rp, raft_pytorch_small as rps

pytestmark = pytest.mark.gpu
F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def T():
    import tf_raft_b200
    from tf_raft_b200 import _lib
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    return tf_raft_b200


@pytest.fixture(scope='module')
def ckpt():
    return rps.synthetic_small_checkpoint(seed=21)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).cuda()


# --------------------------------------------------------------------------------------------- 1. upflow8 kernel
UP_GRIDS = [(1, 1, 1), (2, 1, 1), (1, 1, 9), (1, 7, 1), (3, 5, 7), (1, 13, 11), (2, 9, 128), (1, 136, 240)]


def _flow(shape, seed, special):
    b, h, w = shape
    rng = np.random.default_rng(seed)
    f = (rng.standard_normal((b, h, w, 2)) * 7).astype(F32)
    if special:
        flat = f.reshape(-1)
        idx = rng.choice(flat.size, size=max(1, flat.size // 17), replace=False)
        flat[idx] = rng.choice(np.array([np.nan, np.inf, -np.inf], F32), idx.size)
    return f


@pytest.mark.parametrize('special', [False, True], ids=['finite', 'nan-inf'])
@pytest.mark.parametrize('shape', UP_GRIDS, ids=lambda s: 'x'.join(map(str, s)))
def test_upflow8_align_corners_bit_exact(T, shape, special):
    from tf_raft_b200.layers.corr import upflow8
    flow = _flow(shape, sum(shape), special)
    got = upflow8(dev(flow), align_corners=True)
    torch.cuda.synchronize()
    got = got.cpu().numpy()
    want = rps.upflow8_emulated(flow)
    nan = np.isnan(want)                               # a NaN's payload and sign are the hardware's, not the value's
    assert np.array_equal(np.isnan(got), nan)
    np.testing.assert_array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))
    # torch's own CUDA kernel, NCHW-contiguous (as RAFT-small's flow is) and channels-last.  Measured on an H100 (torch
    # 2.11): the same NaN and inf outputs, 62-100 % of the finite values bit for bit, the rest within 2 ulps of the
    # output's largest magnitude -- the source positions agree and only the final weighted sums round differently
    # (ATen's are compiled with FMA contraction).  Asserted: the same non-finite outputs, and 4 ulps of that scale.
    fin = np.isfinite(want)
    bound = 4 * float(np.spacing(F32(np.abs(want[fin]).max() if fin.any() else 1)))
    for layout in ('nchw', 'channels-last'):
        x = dev(flow).permute(0, 3, 1, 2)
        x = x.contiguous() if layout == 'nchw' else x
        t = (8 * F.interpolate(x, size=(8 * shape[1], 8 * shape[2]), mode='bilinear', align_corners=True)
             ).permute(0, 2, 3, 1).cpu().numpy()
        assert np.array_equal(fin, np.isfinite(t)) and np.array_equal(nan, np.isnan(t))
        d = np.abs(t[fin].astype(np.float64) - want[fin])
        ulp = np.spacing(np.maximum(np.abs(want[fin]), F32(1.0)).astype(F32)).astype(np.float64)
        worst = float((d / ulp).max()) if d.size else 0.0
        print(f'upflow8 {shape} {"nan-inf" if special else "finite"} vs torch CUDA {layout}: bit for bit on '
              f'{int((d == 0).sum())} of {d.size} finite values, worst {worst:.1f} ulp of max(|v|, 1), '
              f'max-abs {float(d.max()) if d.size else 0.0:.2e} (bound {bound:.2e})')
        assert float(d.max()) <= bound if d.size else True


# --------------------------------------------------------------------------------------------- 2. encoders
ENC_GRIDS = list(cases.ENCODER_GRIDS) + [(64, 64), (96, 128), (448, 512)]
_REF = {}


def _encoder_ref(ckpt, images, prefix, kind, key):
    """fp64 output and the largest 1 / sqrt(var + eps) over the instance norms (the factor by which a norm amplifies an
    error in its input), with the largest of the 8-channel norms (layer1) apart."""
    if key not in _REF:
        x = 2 * (torch.from_numpy(images).double().permute(0, 3, 1, 2) / 255.0) - 1.0
        gains = []

        def hook(t):
            gains.append((t.shape[1], float(torch.rsqrt(t.var(dim=(2, 3), unbiased=False) + 1e-5).max())))
        with torch.no_grad():
            out = rps.small_encoder(rp._sd(ckpt, torch.float64), x, prefix, kind, on_norm=hook)
        gain = max([1.0] + [g for _, g in gains])
        gain8 = max([1.0] + [g for c, g in gains if c == 8])
        _REF[key] = out.permute(0, 2, 3, 1).numpy(), gain, gain8
    return _REF[key]


@pytest.mark.parametrize('backend', ['native', 'torch'])
@pytest.mark.parametrize('norm', ['instance', None], ids=['fnet-instance', 'cnet-none'])
@pytest.mark.parametrize('HW', ENC_GRIDS, ids=lambda v: f'{v[0]}x{v[1]}')
def test_bottleneck_encoders_against_fp64(T, ckpt, backend, norm, HW):
    H, W = HW
    if norm == 'instance' and (H, W) == (8, 8):
        pytest.skip('a 1x1 last stage: nn.InstanceNorm2d itself refuses one pixel, so PyTorch RAFT has no value here')
    params = T.load_pytorch_checkpoint(ckpt)
    prefix, out_dim = ('fnet', 128) if norm == 'instance' else ('cnet', 160)
    enc = T.SmallEncoder(output_dim=out_dim, norm_type=norm, backend=backend, conventions='pytorch', blocks='bottleneck',
                         device='cuda')
    enc.load_params(params, prefix + '.')
    im, _ = cases.images(2, H, W)
    got = enc(dev(im), training=False, raw_image=True)
    torch.cuda.synchronize()
    want, gain, gain8 = _encoder_ref(ckpt, im, prefix, norm or 'none', (H, W, norm))
    err = float(np.abs(got.cpu().numpy() - want).max())
    scale = max(1.0, float(np.abs(want).max()))
    print(f'{backend} {norm} {H}x{W}: max-abs {err:.2e} (max |ref| {scale:.2f}, norm gain {gain:.1f}, '
          f'8-channel norms {gain8:.1f})')
    assert err <= 2e-4 * scale * max(1.0, gain / 8)
    if backend == 'native':                            # each image bit for bit independent of its batch
        one = enc(dev(im[1:]), training=False, raw_image=True)
        assert torch.equal(one[0], got[1])


@pytest.mark.parametrize('HW', [(64, 96), (195, 129)], ids=lambda v: f'{v[0]}x{v[1]}')
def test_encode_pair_equals_the_separate_calls(T, ckpt, tmp_path, HW):
    H, W = HW
    m = _model(T, ckpt, tmp_path, 'f16x2')
    im1, im2 = cases.images(2, H, W)
    a, b = dev(im1), dev(im2)
    fmap1, fmap2, net, inp = m._encode_pair(a, b)
    f1, f2 = m.fnet([a, b], training=False, raw_image=True)
    n2, i2 = m._context(a, False)
    torch.cuda.synchronize()
    for x, y in ((fmap1, f1), (fmap2, f2), (net, n2), (inp, i2)):
        assert torch.equal(x, y)


# --------------------------------------------------------------------------------------------- 3. the model
def _model(T, ckpt, tmp_path, precision, **kw):
    path = tmp_path / 'raft-small-synthetic.pth'
    torch.save(ckpt, path)
    m = T.SmallRAFT(conventions='pytorch', blocks='bottleneck', precision=precision, device='cuda', **kw)
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
    preds, low = rps.forward_small(ckpt, im1, im2, iters, flow_init)
    got = got.cpu().numpy()
    # The original's upsampling samples the low-resolution flow at float32 source positions (ATen's align-corners
    # arithmetic), which this model computes as it does, so the gate applies against the fp64 low-resolution flow
    # interpolated at those positions.  Against the all-fp64 F.interpolate the positions' own rounding adds up to
    # 8 * (largest neighbour difference) * 2 ulp(max(h, w)) -- reported, and bounded by that.
    # The gate is 1e-3 for flows up to 128 px and grows in proportion beyond (fp32 rounding grows with the magnitude):
    # the warm-started 440x1024 case reaches 143 px and measured 1.07e-3 (f16x2), the others stay under 1e-3.
    err = np.abs(got - rps.upflow8_fp32_positions(low))
    err64 = np.abs(got - preds[-1])
    diff = max(float(np.abs(np.diff(low, axis=a)).max()) for a in (1, 2))
    pos = 8 * diff * 2 * float(np.spacing(F32(max(H, W) // 8)))
    mag = float(np.abs(preds[-1]).max())
    gate = 1e-3 * max(1.0, mag / 128)
    print(f'{name}: worst final-flow error vs fp64 at the fp32 upsampling positions {err.max():.3e} (gate {gate:.2e}), '
          f'vs all-fp64 {err64.max():.3e} (position allowance {pos:.2e}; |flow| max {mag:.2f})')
    assert err.max() <= gate
    assert err64.max() <= gate + pos


@pytest.mark.parametrize('precision', ['f16x2', 'fp32'])
@pytest.mark.parametrize('grid', [(9, 128), (13, 11)], ids=lambda g: f'{g[0]}x{g[1]}')
def test_fused_loop_equals_the_public_ops(T, ckpt, tmp_path, grid, precision):
    """raft_b200_forward_loop_ex(RAFT_VARIANT_SMALL_PYTORCH, ..., RAFT_SAMPLER_GRID) gives, byte for byte, what the loop
    spelled out with CorrBlock(sampler='grid_sample').retrieve, update_block and upflow8(align_corners=True) gives, at
    every iteration and with last_only=True."""
    from tf_raft_b200.layers.corr import upflow8
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
        net, _, delta = model.update_block([net, inp, corr, coords1 - grid0])
        coords1 = coords1 + delta
        ups.append(upflow8(coords1 - grid0, align_corners=True))
        assert torch.equal(ups[-1], model.upsample_flow(coords1 - grid0))
    full = model([a, b], training=False)
    assert len(full) == iters
    for i in range(iters):
        assert torch.equal(full[i], ups[i]), f'iteration {i}: max-abs {float((full[i] - ups[i]).abs().max()):.3e}'
    last = model([a, b], training=False, last_only=True)
    assert len(last) == 1 and torch.equal(last[0], ups[-1]), 'last_only differs from the loop spelled out'


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
    warm = [f.clone() for f in m.predict_video(frames)]
    assert torch.equal(warm[0], video[0])


# --------------------------------------------------------------------------------------------- 4. guards
def test_guards(T, ckpt, tmp_path):
    import ctypes
    from tf_raft_b200 import _lib
    with pytest.raises(ValueError, match='bottleneck'):
        T.SmallRAFT(conventions='pytorch', device='cuda')
    with pytest.raises(ValueError, match='bottleneck'):
        T.SmallRAFT(blocks='bottleneck', device='cuda')
    with pytest.raises(TypeError, match='blocks'):
        T.RAFT(conventions='pytorch', blocks='bottleneck', device='cuda')
    with pytest.raises(ValueError):
        T.SmallEncoder(output_dim=128, norm_type='batch', conventions='pytorch', blocks='bottleneck', device='cuda')
    with pytest.raises(ValueError):
        T.BasicEncoder(output_dim=128, norm_type='instance', conventions='pytorch', blocks='bottleneck', device='cuda')
    m = _model(T, ckpt, tmp_path, 'f16x2')
    with pytest.raises(NotImplementedError):
        m.compile(optimizer=T.TorchAdamW(1e-4, 1e-4))
    with pytest.raises(NotImplementedError):
        m.train_step(None)
    basic = tmp_path / 'raft-basic.pth'
    torch.save(rp.synthetic_checkpoint(seed=2), basic)
    with pytest.raises(ValueError, match='RAFT-small'):
        m.load_pytorch_weights(str(basic))
    small = tmp_path / 'raft-small-synthetic.pth'
    with pytest.raises(ValueError, match='RAFT-small'):
        T.RAFT(conventions='pytorch', device='cuda').load_pytorch_weights(str(small))
    # the library: entry points other than the encoders' and the loop's refuse the variant
    L = _lib.lib()
    v = _lib.VARIANT_SMALL_PYTORCH
    n = ctypes.c_size_t()
    assert L.raft_b200_update_prepared_bytes(v, 196, 1, ctypes.byref(n)) == -1
    assert L.raft_b200_update_workspace_bytes(v, 1, 8, 8, 1, ctypes.byref(n)) == -1
    assert L.raft_b200_encoder_prepared_bytes(v, 128, ctypes.byref(n)) == 0 and n.value > 0
    assert L.raft_b200_encoder_workspace_bytes(v, 1, 64, 64, ctypes.byref(n)) == 0 and n.value > 0
    blob = torch.empty(1 << 20, dtype=torch.uint8, device='cuda')
    w = _lib.RaftEncoderWeights()
    assert L.raft_b200_encoder_prepare_ex(v, 1, 128, ctypes.byref(w), 1, _lib.ptr(blob), blob.numel(), None) == -1
    bw = _lib.RaftBottleneckEncoderWeights()
    assert L.raft_b200_encoder_prepare_bottleneck(2, 128, ctypes.byref(bw), _lib.ptr(blob), blob.numel(), None) == -1
    assert L.raft_b200_encoder_forward(v, 2, 128, _lib.ptr(blob), _lib.ptr(blob), 1, 64, 64, 0, 1, _lib.ptr(blob),
                                       _lib.ptr(blob), blob.numel(), None) == -1
    odd = torch.empty(64, device='cuda')
    assert L.raft_b200_upflow8_align_corners(_lib.ptr(odd[1:]), 1, 2, 2, _lib.ptr(odd), None) == -1


# --------------------------------------------------------------------------------------------- 5. evaluate.py
def test_evaluate_script_scores_raft_small(T, ckpt, tmp_path):
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import test_gpu_pad as gp
    root = str(tmp_path / 'data')
    gp._write_trees(root)
    path = tmp_path / 'raft-small-synthetic.pth'
    torch.save(ckpt, path)
    res = gp._script('evaluate.py', 'sintel', '--root', os.path.join(root, 'sintel'), '--pytorch-checkpoint', str(path),
                     '--small', '--iters', '3', '--workers', '2')
    assert res['conventions'] == 'pytorch' and res['padding'] == 'replicate' and res['iters'] == 3
    assert res['pixels'] == 2 * 60 * 90 + 3 * 61 * 84 and res['pairs'] == 5
    # the same score in process
    m = _model(T, ckpt, tmp_path, 'f16x2', iters_pred=3)
    want = T.evaluate(m, gp._dataset(root, 'sintel'), batch_size=4, max_flow=None, protocol='pixel', workers=2,
                      padding='replicate', pad_mode='sintel')
    assert res['epe'] == pytest.approx(want['epe'], rel=1e-6)
