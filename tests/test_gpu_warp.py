"""Flow warping, flow composition and RAFT.track_video on the GPU.

The kernels (raft_b200_warp, raft_b200_compose_flow) equal the NumPy float32 restatement (oracle.warp_np) bit for bit
at every shape class, channel count, mode, dtype and edge landing; labels come through unchanged; results do not
depend on the batch; graph capture replays the eager calls; host-side argument checks launch nothing; track_video is
the restatement's chaining of predict_video(bidirectional=True)'s own yields, for RAFT and RAFT(conventions='pytorch').
"""
import ctypes

import numpy as np
import pytest
import torch

import cases
from oracle import raft_pytorch as rp, warp_np, weights
from test_warp_ref import flow_case, texels

F32 = np.float32


@pytest.fixture(scope='module')
def T():
    import tf_raft_b200
    from tf_raft_b200 import _lib
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    return tf_raft_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits_equal(got, want, what=''):
    got = got.cpu().numpy()
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    if got.dtype == F32:
        nan = np.isnan(want)                           # a NaN's payload and sign are the hardware's, not the value's
        np.testing.assert_array_equal(np.isnan(got), nan, err_msg=what)
        got, want = got[~nan].view(np.int32), want[~nan].view(np.int32)
    np.testing.assert_array_equal(got, want, err_msg=what)


# --------------------------------------------------------------------------------------------- warp, bit for bit
GRIDS = [(1, 1, 1, 1, 1), (2, 1, 37, 1, 37), (2, 29, 1, 29, 1), (3, 7, 13, 7, 13), (2, 9, 15, 20, 6),
         (1, 436, 1024, 436, 1024), (1, 1080, 1920, 1080, 1920)]


@pytest.mark.gpu
@pytest.mark.parametrize('grid', GRIDS, ids=lambda g: 'x'.join(map(str, g)))
@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
def test_warp_bit_exact_float32(T, grid, mode):
    b, h, w, hs, ws = grid
    flow = flow_case(b, h, w, 11, hs, ws)
    for c in ((1, 3) if h * w > 10000 else (1, 2, 3, 16)):
        src = texels(b, hs, ws, c, 12 + c, nonfinite=True)
        want, want_occ = warp_np.warp(src, flow, mode, fill=-1.5)
        got, occ = T.warp(dev(src), dev(flow), mode=mode, fill=-1.5)
        _bits_equal(got, want, f'{mode} C={c}')
        _bits_equal(occ, want_occ)
        assert occ.dtype == torch.bool


@pytest.mark.gpu
@pytest.mark.parametrize('c', [64, 1024])
@pytest.mark.parametrize('mode', ['bilinear', 'nearest'])
def test_warp_bit_exact_wide_channels(T, c, mode):
    b, h, w = 2, 11, 17
    flow = flow_case(b, h, w, 21, 9, 23)
    src = texels(b, 9, 23, c, 22, nonfinite=True)
    want, want_occ = warp_np.warp(src, flow, mode)
    got, occ = T.warp(dev(src), dev(flow), mode=mode)
    _bits_equal(got, want)
    _bits_equal(occ, want_occ)


@pytest.mark.gpu
@pytest.mark.parametrize('grid', GRIDS, ids=lambda g: 'x'.join(map(str, g)))
def test_warp_uint8_nearest_bit_exact_and_labels_preserved(T, grid):
    b, h, w, hs, ws = grid
    rng = np.random.default_rng(31)
    labels = rng.choice(np.array([3, 17, 200, 254], np.uint8), (b, hs, ws, 1))
    flow = flow_case(b, h, w, 32, hs, ws)
    want, want_occ = warp_np.warp(labels, flow, 'nearest', fill=255)
    got, occ = T.warp(dev(labels), dev(flow), mode='nearest', fill=255)
    _bits_equal(got, want)
    _bits_equal(occ, want_occ)
    present = set(np.unique(labels).tolist())
    assert set(np.unique(got[~occ].cpu().numpy()).tolist()) <= present
    assert (got[occ] == 255).all()


@pytest.mark.gpu
def test_warp_batch_independence(T):
    b, h, w, c = 4, 31, 45, 5
    flow, src = flow_case(b, h, w, 41), texels(b, h, w, c, 42, nonfinite=True)
    for mode in ('bilinear', 'nearest'):
        out, occ = T.warp(dev(src), dev(flow), mode=mode)
        for i in range(b):
            one, one_occ = T.warp(dev(src[i:i + 1]), dev(flow[i:i + 1]), mode=mode)
            assert torch.equal(out[i:i + 1].view(torch.int32), one.view(torch.int32)) and torch.equal(occ[i:i + 1], one_occ)
    f2 = flow_case(b, h, w, 43)
    acc, lost = T.compose_flow(dev(flow), dev(f2))
    for i in range(b):
        one, one_lost = T.compose_flow(dev(flow[i:i + 1]), dev(f2[i:i + 1]))
        assert torch.equal(acc[i:i + 1].view(torch.int32), one.view(torch.int32)) and torch.equal(lost[i:i + 1], one_lost)


# --------------------------------------------------------------------------------------------- compose, bit for bit
@pytest.mark.gpu
@pytest.mark.parametrize('grid', [(1, 1, 1), (2, 1, 37), (2, 29, 1), (3, 7, 13), (1, 436, 1024), (1, 1080, 1920)],
                         ids=lambda g: 'x'.join(map(str, g)))
@pytest.mark.parametrize('masks', ['none', 'occ1', 'occ2', 'both'])
def test_compose_bit_exact(T, grid, masks):
    b, h, w = grid
    rng = np.random.default_rng(51)
    f1 = flow_case(b, h, w, 52)
    f2 = texels(b, h, w, 2, 53, nonfinite=True)
    occ1 = rng.random((b, h, w)) < 0.2 if masks in ('occ1', 'both') else None
    occ2 = rng.random((b, h, w)) < 0.2 if masks in ('occ2', 'both') else None
    want, want_occ = warp_np.compose_flow(f1, f2, occ1, occ2)
    got, occ = T.compose_flow(dev(f1), dev(f2), None if occ1 is None else dev(occ1), None if occ2 is None else dev(occ2))
    _bits_equal(got, want)
    _bits_equal(occ, want_occ)
    assert torch.isfinite(got[~occ]).all()


@pytest.mark.gpu
def test_compose_in_place_aliases(T, L):
    """out may be f1 and occ_out may be occ1: the in-place call equals the out-of-place one."""
    from tf_raft_b200 import _lib
    b, h, w = 2, 33, 47
    f1, f2 = dev(flow_case(b, h, w, 61)), dev(texels(b, h, w, 2, 62))
    occ1 = dev(np.random.default_rng(63).random((b, h, w)) < 0.3).view(torch.uint8)
    want, want_occ = T.compose_flow(f1, f2, occ1)
    _lib.call('compose_flow', f1.device, _lib.ptr(f1), _lib.ptr(f2), _lib.ptr(occ1), None, b, h, w, _lib.ptr(f1),
              _lib.ptr(occ1))
    assert torch.equal(f1.view(torch.int32), want.view(torch.int32)) and torch.equal(occ1.bool(), want_occ)


# --------------------------------------------------------------------------------------------- graphs and arguments
@pytest.mark.gpu
def test_graph_capture_equals_eager(T):
    b, h, w, c = 2, 64, 96, 3
    src, flow, f2 = dev(texels(b, h, w, c, 71)), dev(flow_case(b, h, w, 72)), dev(texels(b, h, w, 2, 73))
    want = T.warp(src, flow) + T.compose_flow(flow, f2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                     # warm the allocator outside the capture
        T.warp(src, flow), T.compose_flow(flow, f2)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = T.warp(src, flow) + T.compose_flow(flow, f2)
    src.mul_(2)
    g.replay()
    torch.cuda.synchronize()
    want2 = T.warp(src, flow)
    assert torch.equal(got[0], want2[0]) and torch.equal(got[1], want2[1])
    assert torch.equal(got[2].view(torch.int32), want[2].view(torch.int32)) and torch.equal(got[3], want[3])


@pytest.fixture(scope='module')
def L(T):
    from tf_raft_b200 import _lib
    return _lib.lib()


@pytest.mark.gpu
def test_argument_errors_launch_nothing(T, L):
    from tf_raft_b200 import _lib
    buf = torch.empty(1 << 20, dtype=torch.uint8, device='cuda')
    base = buf.data_ptr()
    a, bb, c, d = (ctypes.c_void_p(base + k * (1 << 18)) for k in range(4))
    odd = ctypes.c_void_p(base + 4)
    odd1 = ctypes.c_void_p(base + (1 << 18) + 1)
    warp, comp = L.raft_b200_warp, L.raft_b200_compose_flow
    ok = dict(src=a, dtype=0, Hs=8, Ws=8, C=3, flow=bb, B=1, H=8, W=8, mode=0, fill=0.0, out=c, occ=d)

    def w(**kw):
        args = dict(ok, **kw)
        return warp(*args.values(), None)

    _lib.launch_count_reset()
    bad_arg = [dict(src=None), dict(flow=None), dict(out=None), dict(mode=2), dict(mode=-1), dict(dtype=2),
               dict(dtype=1, mode=0), dict(dtype=1, mode=1, fill=256.0), dict(dtype=1, mode=1, fill=1.5),
               dict(dtype=1, mode=1, fill=-1.0), dict(dtype=1, mode=1, fill=float('nan')), dict(flow=odd),
               dict(src=odd1), dict(out=odd1), dict(out=a), dict(out=bb), dict(occ=a), dict(occ=bb), dict(occ=c),
               dict(out=ctypes.c_void_p(base + 64))]
    for kw in bad_arg:
        assert w(**kw) == -1, kw
    for kw in (dict(B=0), dict(H=0), dict(W=-1), dict(Hs=0), dict(Ws=0), dict(C=0), dict(C=1025),
               dict(H=1 << 16, W=1 << 13, C=4), dict(Hs=1 << 16, Ws=1 << 13, C=4)):
        assert w(**kw) == -2, kw
    assert w(dtype=1, mode=1, fill=255.0, src=odd1, out=ctypes.c_void_p(base + 3 * (1 << 18) + 1), occ=None) == 0
    torch.cuda.synchronize()
    assert _lib.launch_count() == 1

    _lib.launch_count_reset()
    f1, f2, o1, o2, out, oo = (ctypes.c_void_p(base + k * (1 << 17)) for k in range(6))
    okc = dict(f1=f1, f2=f2, occ1=o1, occ2=o2, B=1, H=8, W=8, out=out, occ_out=oo)

    def cp(**kw):
        args = dict(okc, **kw)
        return comp(*args.values(), None)

    for kw in (dict(f1=None), dict(f2=None), dict(out=None), dict(occ_out=None), dict(f1=odd), dict(f2=odd),
               dict(out=odd), dict(out=f2), dict(out=ctypes.c_void_p(base + 8)), dict(out=o1), dict(out=o2),
               dict(occ_out=f1), dict(occ_out=f2), dict(occ_out=o2), dict(occ_out=out),
               dict(occ_out=ctypes.c_void_p(base + (1 << 17) * 2 + 1))):
        assert cp(**kw) == -1, kw
    for kw in (dict(B=0), dict(H=-1), dict(W=0), dict(H=1 << 16, W=1 << 15)):
        assert cp(**kw) == -2, kw
    assert _lib.launch_count() == 0
    assert cp(out=f1, occ_out=o1, occ2=None) == 0
    torch.cuda.synchronize()
    assert _lib.launch_count() == 1


@pytest.mark.gpu
def test_python_argument_errors(T):
    f = torch.zeros((2, 8, 12, 2), device='cuda')
    src = torch.zeros((2, 8, 12, 3), device='cuda')
    with pytest.raises(TypeError):
        T.warp(np.zeros((2, 8, 12, 3), F32), f)
    with pytest.raises(TypeError):
        T.warp(src.int(), f)
    with pytest.raises(ValueError):
        T.warp(src, f, mode='bicubic')
    with pytest.raises(ValueError):
        T.warp(src.to(torch.uint8), f)                               # bilinear on labels
    with pytest.raises(ValueError):
        T.warp(src.to(torch.uint8), f, mode='nearest', fill=300)
    with pytest.raises(ValueError):
        T.warp(src[:1], f)
    with pytest.raises(ValueError):
        T.warp(src[..., 0], f)
    with pytest.raises(ValueError):
        T.warp(torch.zeros((2, 8, 12, 1025), device='cuda'), f)
    with pytest.raises(ValueError):
        T.warp(src, f[..., :1])
    with pytest.raises(ValueError):
        T.compose_flow(f, f[:1])
    with pytest.raises(TypeError):
        T.compose_flow(f, f, occ1=torch.zeros((2, 8, 12), device='cuda'))
    with pytest.raises(ValueError):
        T.compose_flow(f, f, occ2=torch.zeros((2, 8, 11), dtype=torch.bool, device='cuda'))
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        T.warp(src.cpu(), f.cpu())
    out, occ = T.warp(src.double(), f)
    assert out.dtype == torch.float32 and occ.dtype == torch.bool


# --------------------------------------------------------------------------------------------- track_video
def _clip(bs, n, H, W, seed=90):
    """Textured frames with a dark square occluder moving 5 px per frame across them."""
    frames = []
    for t in range(n):
        im = cases.images(bs, H, W, seed, seed)[0].copy()
        im = np.roll(im, 2 * t, axis=2)                                    # a slow pan of the texture
        im[:, 20:40, 10 + 5 * t:30 + 5 * t] = 16.0
        frames.append(dev(im.astype(F32)))
    return frames


def _models(T, tmp_path):
    p = weights.init_params('raft', 1234, bias_scale=0.05, norm_jitter=0.1)
    tf = T.RAFT(iters=3, iters_pred=3, precision='f16x2')
    tf.load_params(p)
    path = tmp_path / 'raft-synthetic.pth'
    torch.save(rp.synthetic_checkpoint(seed=7), path)
    pt = T.RAFT(iters=3, iters_pred=3, conventions='pytorch', precision='f16x2', device='cuda')
    pt.load_pytorch_weights(str(path))
    return {'tf-raft': tf, 'pytorch': pt}


@pytest.mark.gpu
@pytest.mark.parametrize('warm_start', [True, False], ids=['warm', 'cold'])
def test_track_video_is_the_chain_of_predict_video(T, tmp_path, warm_start):
    bs, n, H, W = 2, 5, 64, 96
    frames = _clip(bs, n, H, W)
    for name, model in _models(T, tmp_path).items():
        pairs = [tuple(x.clone() for x in y) for y in model.predict_video(iter(frames), warm_start=warm_start,
                                                                          bidirectional=True)]
        assert len(pairs) == n - 1
        fw = [p[0].cpu().numpy() for p in pairs]
        bw = [p[1].cpu().numpy() for p in pairs]
        ofw = [p[2].cpu().numpy() for p in pairs]
        obw = [p[3].cpu().numpy() for p in pairs]
        for direction, want in (('forward', warp_np.track_forward(fw, ofw)),
                                ('backward', warp_np.track_backward(bw, obw))):
            got = list(model.track_video(iter(frames), direction=direction, warm_start=warm_start))
            assert len(got) == n - 1
            for t, ((flow, occ), (wf, wo)) in enumerate(zip(got, want), start=1):
                assert tuple(flow.shape) == (bs, H, W, 2) and occ.dtype == torch.bool
                _bits_equal(flow, wf, f'{name} {direction} t={t}')
                _bits_equal(occ, wo, f'{name} {direction} t={t}')
            lost = [o.cpu().numpy() for _, o in got]
            assert all((b >= a).all() for a, b in zip(lost, lost[1:]))
        again = list(model.predict_video(iter(frames), warm_start=warm_start, bidirectional=True))
        for p, q in zip(pairs, again):
            assert all(torch.equal(x, y) for x, y in zip(p, q)), name


@pytest.mark.gpu
def test_track_video_guards(T):
    model = T.SmallRAFT(iters=2, iters_pred=2)
    frames = _clip(1, 3, 64, 96)
    got = list(model.track_video(frames, direction='backward'))
    assert len(got) == 2 and tuple(got[0][0].shape) == (1, 64, 96, 2)
    assert list(model.track_video(frames[:1])) == []
    with pytest.raises(ValueError):
        list(model.track_video(frames, direction='sideways'))
    with pytest.raises(ValueError):
        list(model.track_video([frames[0], frames[1][:, :56]]))
    model.iters_pred = 0
    with pytest.raises(ValueError):
        list(model.track_video(frames))
