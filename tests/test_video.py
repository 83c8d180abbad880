"""Video inference: RAFT's warm start and `predict_video`, which encodes every frame once.

The warm start carries a pair's low-resolution flow to the next pair by forward interpolation
(raft_b200_forward_interpolate, `forward_interpolate`) and enters the loop at coords0 + flow_init
(raft_b200_coords_init, `RAFT.__call__(..., flow_init=...)`).  CPU: the NumPy restatement (oracle.video_np) against
scipy's griddata, the oracle's warm-start forward (oracle.warm_start) against oracle.raft_torch, host-side argument
checks.  GPU: the kernels bit for bit against NumPy, zero warm start == cold start, warm start against the fp64 oracle,
the fused loop against the public ops from a warm state, CUDA-graph replay with flow_init, and the video generator
against per-pair calls and against the oracle.
"""
import ctypes

import numpy as np
import pytest
import torch

import cases
from oracle import raft_torch as rt, video_np, warm_start, weights

F32 = np.float32
PRECISIONS = ('f16x2', 'fp32')


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _cls(T, variant):
    return T.RAFT if variant == 'raft' else T.SmallRAFT


@pytest.fixture(scope='module')
def L():
    from tf_raft_b200 import build, _lib
    build.build()
    return _lib.lib()


@pytest.fixture(scope='module')
def T():
    import tf_raft_b200
    from tf_raft_b200 import _lib
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    return tf_raft_b200


# --------------------------------------------------------------------------------------------- seeded flows
def _plant(flat, rng, h, w):
    """NaN / +-inf sources, then pairs of sources whose integer flows land on the same integer point strictly inside
    the frame (exact ties: the lower index must win)."""
    n = h * w
    k = max(1, n // 50)
    sel = rng.choice(n, size=min(n, 3 * k), replace=False)
    flat[sel[:k], 0] = np.nan
    flat[sel[k:2 * k], 1] = np.inf
    flat[sel[2 * k:], 0] = -np.inf
    if h >= 3 and w >= 3 and n >= 2:
        for _ in range(k):
            i, j = rng.choice(n, 2, replace=False)
            px, py = rng.integers(1, w - 1), rng.integers(1, h - 1)
            for s in (i, j):
                flat[s] = (px - s % w, py - s // w)
    return flat


def fi_case(h, w, seed):
    """(3, h, w, 2): image 0 sub-pixel flow (+-0.3 px: most targets have their own source), image 1 pushes every source
    out of the frame (-> zero flow), image 2 large flow (+-20 px: holes) with a quarter of it integer; NaN, +-inf and
    planted exact ties in images 0 and 2."""
    rng = np.random.default_rng(seed)
    f = np.empty((3, h, w, 2), F32)
    f[0] = rng.uniform(-0.3, 0.3, (h, w, 2))
    f[1, ..., 0] = w + rng.uniform(0, 5, (h, w))
    f[1, ..., 1] = rng.uniform(-20, 20, (h, w))
    f[2] = rng.uniform(-20, 20, (h, w, 2))
    flat2 = f[2].reshape(-1, 2)
    flat2[::4] = np.round(flat2[::4])
    _plant(f[0].reshape(-1, 2), rng, h, w)
    _plant(flat2, rng, h, w)
    return f


def smooth_flow(b, h, w, amp=2.5, seed=0):
    """A smooth, non-integer flow of a few pixels (B, h, w, 2)."""
    rng = np.random.default_rng(seed)
    gy, gx = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing='ij')
    out = np.empty((b, h, w, 2), F32)
    for k in range(b):
        p = rng.uniform(0, 2 * np.pi, 4)
        out[k, ..., 0] = 0.37 + amp * np.sin(2 * np.pi * gx / w + p[0]) * np.cos(2 * np.pi * gy / h + p[1])
        out[k, ..., 1] = -0.21 + amp * np.cos(2 * np.pi * gx / w + p[2]) * np.sin(2 * np.pi * gy / h + p[3])
    return out


# --------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize('kind', ['subpixel', 'holes', 'integer', 'special'])
def test_numpy_forward_interpolate_is_griddata_nearest(kind):
    """oracle.video_np.forward_interpolate is scipy.interpolate.griddata((x1, y1), f, (X, Y), method='nearest') over the
    sources landing strictly inside the frame -- RAFT's forward interpolation -- up to the tie rule: wherever griddata
    picks another source than the restatement, the two sources' fp64 distances tie.  An image with no valid source,
    where griddata has nothing to interpolate from, gets zero flow."""
    from scipy.interpolate import griddata
    b, h, w = 3, 13, 17
    rng = np.random.default_rng({'subpixel': 1, 'holes': 2, 'integer': 3, 'special': 4}[kind])
    if kind == 'subpixel':
        flow = rng.uniform(-0.3, 0.3, (b, h, w, 2)).astype(F32)
    elif kind == 'holes':
        flow = rng.uniform(-20, 20, (b, h, w, 2)).astype(F32)
    elif kind == 'integer':                                  # exact integer landings: ties everywhere
        flow = rng.integers(-5, 6, (b, h, w, 2)).astype(F32)
    else:
        flow = fi_case(h, w, 5)
    out, idx = video_np.forward_interpolate(flow, return_index=True)
    assert out.dtype == F32 and out.shape == flow.shape and np.isfinite(out).all()
    x1, y1, valid = video_np.landing(flow)
    tx = np.tile(np.arange(w, dtype=np.float64), h)
    ty = np.repeat(np.arange(h, dtype=np.float64), w)
    differ = 0
    for k in range(b):
        src = np.nonzero(valid[k])[0]
        if src.size == 0:
            assert not out[k].any() and (idx[k] == -1).all()
            continue
        pick = griddata((x1[k, src], y1[k, src]), src.astype(np.float64), (tx, ty), method='nearest').astype(np.int64)
        mine = idx[k]
        assert valid[k][mine].all()
        d_mine = (x1[k, mine] - tx) ** 2 + (y1[k, mine] - ty) ** 2
        d_pick = (x1[k, pick] - tx) ** 2 + (y1[k, pick] - ty) ** 2
        assert (d_mine <= d_pick).all(), 'the restatement missed a nearer source'
        tie = pick != mine
        assert (np.abs(d_pick - d_mine)[tie] <= 1e-12 * np.maximum(d_mine, d_pick)[tie]).all()
        assert (mine[tie] < pick[tie]).all(), 'ties go to the lowest source index'
        differ += int(tie.sum())
        np.testing.assert_array_equal(out[k].reshape(-1, 2), flow[k].reshape(-1, 2)[mine])
    if kind == 'special':
        assert not out[1].any()
    if kind == 'integer':
        assert differ > 0, 'integer landings should give griddata ties to break'


@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_oracle_zero_flow_init_is_the_cold_start(variant):
    """oracle.warm_start.forward without a flow_init, and with a zero one, is oracle.raft_torch.forward exactly:
    predictions, per-iteration lookups and coordinates, in fp32 and fp64."""
    p = weights.init_params(variant, 1234, bias_scale=0.05, norm_jitter=0.1)
    im1, im2 = cases.images(2, 64, 96)
    for dtype in (torch.float32, torch.float64):
        cold, ci = rt.forward(p, im1, im2, variant, 2, dtype=dtype, return_intermediates=True)
        for fi in (None, np.zeros((2, 8, 12, 2), F32)):
            warm, wi = warm_start.forward(p, im1, im2, variant, 2, dtype=dtype, flow_init=fi, return_intermediates=True)
            assert len(cold) == len(warm) == 2
            for i in range(2):
                assert torch.equal(cold[i], warm[i])
                assert torch.equal(ci['corr'][i], wi['corr'][i]) and torch.equal(ci['coords'][i], wi['coords'][i])


def test_host_side_argument_errors_of_the_warm_start_entry_points(L):
    """raft_b200_forward_interpolate / raft_b200_coords_init validate on the host like the other entry points: NULL
    pointers -> RAFT_ERR_BAD_ARG, non-positive dims -> RAFT_ERR_BAD_SHAPE, and forward interpolation refuses grids whose
    pixel count does not fit its int indices."""
    fake = ctypes.c_void_p(0x1000)
    for fn in (L.raft_b200_forward_interpolate, L.raft_b200_coords_init):
        assert fn(None, 1, 8, 8, fake, None) == -1
        assert fn(fake, 1, 8, 8, None, None) == -1
        assert fn(fake, 0, 8, 8, fake, None) == -2
        assert fn(fake, 1, -3, 8, fake, None) == -2
        assert fn(fake, 1, 8, 0, fake, None) == -2
    assert L.raft_b200_forward_interpolate(fake, 1, 65536, 32768, fake, None) == -2     # h*w = 2^31
    assert L.raft_b200_forward_interpolate(fake, 1, 46341, 46341, fake, None) == -2     # h*w > 2^31 - 1
    assert L.raft_b200_forward_interpolate(fake, 1, 1, (1 << 31) - 100, fake, None) == -2      # within 512 of 2^31
    assert L.raft_b200_abi_version() == 2


# --------------------------------------------------------------------------------------------- GPU: the kernels
FI_GRIDS = [(1, 1), (7, 5), (56, 64), (56, 128)] + [(h, w) for _, h, w in cases.TILE_GRIDS] + [(216, 216)]


@pytest.mark.gpu
@pytest.mark.parametrize('grid', FI_GRIDS, ids=lambda g: f'{g[0]}x{g[1]}')
def test_forward_interpolate_bit_exact(T, grid):
    """The CUDA kernel equals the NumPy fp64 brute force bit for bit, batch 3: sub-pixel flow, an image pushed entirely
    out of the frame (zero flow), large flow with holes, NaN and +-inf sources (never chosen, never emitted) and
    planted exact ties (the lower source index)."""
    h, w = grid
    flow = fi_case(h, w, 1000 * h + w)
    want = video_np.forward_interpolate(flow)
    got = T.forward_interpolate(dev(flow))
    assert got.dtype == torch.float32 and tuple(got.shape) == flow.shape
    got = got.cpu().numpy()
    np.testing.assert_array_equal(got, want)
    assert np.isfinite(got).all() and not got[1].any()
    with pytest.raises(ValueError):
        T.forward_interpolate(dev(flow[..., :1]))


@pytest.mark.gpu
def test_coords_init_bit_exact(T):
    """raft_b200_coords_init = coords_grid + flow_init with one fp32 rounding per component (NumPy float32)."""
    from tf_raft_b200.layers.corr import coords_init
    rng = np.random.default_rng(8)
    for b, h, w in ((3, 7, 5), (2, 56, 128), (1, 216, 216)):
        flow = (rng.standard_normal((b, h, w, 2)) * 30).astype(F32)
        flat = flow.reshape(-1, 2)
        flat[::7] = rng.uniform(-1e-6, 1e-6, flat[::7].shape)        # below half an ulp of the grid: rounds away
        flat[1::11] = np.round(flat[1::11])
        flat[2::13, 0] = np.nan
        flat[3::17, 1] = -np.inf
        gy, gx = np.meshgrid(np.arange(h, dtype=F32), np.arange(w, dtype=F32), indexing='ij')
        want = np.stack([gx, gy], axis=-1)[None] + flow
        np.testing.assert_array_equal(coords_init(dev(flow)).cpu().numpy(), want)


# --------------------------------------------------------------------------------------------- GPU: warm start
def _model(T, variant, precision, params, iters, **kw):
    model = _cls(T, variant)(iters=iters, iters_pred=iters, precision=precision, **kw)
    model.load_params(params)
    return model


@pytest.mark.gpu
@pytest.mark.parametrize('use_graph', [False, True], ids=['eager', 'graph'])
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_zero_warm_start_is_the_cold_start(T, variant, precision, use_graph):
    p = weights.init_params(variant, 1234, bias_scale=0.05, norm_jitter=0.1)
    im1, im2 = cases.images(2, 64, 96)
    a, b = dev(im1), dev(im2)
    model = _model(T, variant, precision, p, 3, use_graph=use_graph)
    for last_only in (False, True):
        for _ in range(2 if use_graph else 1):                   # capture, then a pure replay
            cold = [t.clone() for t in model([a, b], training=False, last_only=last_only)]
            warm = [t.clone() for t in model([a, b], training=False, last_only=last_only,
                                             flow_init=torch.zeros((2, 8, 12, 2), device='cuda'))]
            assert len(cold) == len(warm) == (1 if last_only else 3)
            for i, (c, w) in enumerate(zip(cold, warm)):
                assert torch.equal(c, w), f'prediction {i}, last_only={last_only}'


@pytest.mark.gpu
def test_flow_init_argument_errors(T):
    model = T.RAFT(iters=1, iters_pred=1)
    im1, im2 = cases.images(2, 64, 96)
    a, b = dev(im1), dev(im2)
    with pytest.raises(ValueError):
        model([a, b], training=False, flow_init=torch.zeros((2, 8, 11, 2), device='cuda'))
    with pytest.raises(ValueError):
        model([a, b], training=False, flow_init=torch.zeros((1, 8, 12, 2), device='cuda'))
    with pytest.raises(ValueError):
        model([a, b], training=False, flow_init=torch.zeros((2, 8, 12, 2)))             # CPU
    with pytest.raises(TypeError):
        model([a, b], training=False, flow_init=torch.zeros((2, 8, 12, 2), dtype=torch.float64, device='cuda'))
    with pytest.raises(TypeError):
        model([a, b], training=False, flow_init=np.zeros((2, 8, 12, 2), F32))


def _sampler_flips(inter, gpu_coords, i, radius):
    """Taps where the ORACLE sampler, evaluated on the oracle pyramid, gives a different branch of its discontinuity
    (integer / border => 0, corr.py:45-60) for the GPU's coordinates than for the oracle's (as in
    test_gpu_parity.test_raft_448x512_final_flow, for either radius)."""
    cb = rt.CorrBlock.__new__(rt.CorrBlock)
    cb.corr_pyramid, cb.num_levels, cb.radius = inter['corr_pyramid'], 4, radius
    at_gpu = cb.retrieve(gpu_coords.cpu().to(inter['corr'][i].dtype))
    return int(((at_gpu - inter['corr'][i]).abs() > 0.5).sum())


def _spelled_out(T, model, a, b, flow_init, iters):
    """The loop spelled out with the public ops from coords0 + flow_init: (coords1 entering every iteration, the
    prediction of every iteration, coords1 after the last)."""
    fmap1, fmap2, net, inp = model._encode(a, b, False)
    cb = T.CorrBlock(fmap1, fmap2, model.corr_levels, model.corr_radius, precision=model.precision)
    bs, h, w, _ = fmap1.shape
    grid0 = T.coords_grid(bs, h, w)
    coords1 = grid0.clone() if flow_init is None else grid0 + flow_init
    coords, ups = [], []
    for _ in range(iters):
        coords.append(coords1)
        corr = cb.retrieve(coords1)
        net, mask, delta = model.update_block([net, inp, corr, coords1 - grid0])
        coords1 = coords1 + delta
        ups.append(model.upsample_flow(coords1 - grid0, mask))
    return coords, ups, coords1


def _gate(inter, want, coords, ups, radius):
    """(max-abs over the iterations before the first sampler-discontinuity crossing, that iteration or None)."""
    first_flip = None
    for i in range(len(ups)):
        if _sampler_flips(inter, coords[i], i, radius):
            first_flip = i
            break
    n = len(ups) if first_flip is None else first_flip
    worst = max([float((ups[i].cpu().double() - want[i]).abs().max()) for i in range(n)], default=0.0)
    return worst, first_flip


@pytest.mark.gpu
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('variant,shape,iters', [('raft', (72, 200), 3), ('small', (128, 256), 4)])
def test_warm_start_vs_fp64_oracle(T, variant, shape, iters, precision):
    """A smooth, non-integer flow_init of a few pixels: every iteration within 1e-3 max-abs of the fp64 oracle started
    from coords0 + flow_init, up to the first crossing of a discontinuity of the reference sampler (DESIGN.md section
    4).  Weights and images of test_gpu_parity.test_other_resolutions_vs_oracle."""
    H, W = shape
    p = weights.init_params(variant, 77, bias_scale=0.02, norm_jitter=0.05)
    im1, im2 = cases.images(1, H, W, 11, 12)
    fi = smooth_flow(1, H // 8, W // 8, seed=3)
    want, inter = warm_start.forward(p, im1, im2, variant, iters, dtype=torch.float64, flow_init=fi,
                                     return_intermediates=True)
    model = _model(T, variant, precision, p, iters)
    coords, ups, _ = _spelled_out(T, model, dev(im1), dev(im2), dev(fi), iters)
    worst, first_flip = _gate(inter, want, coords, ups, model.corr_radius)
    msg = f'{variant} {precision}: max-abs {worst:.3e} before the first crossing (iteration {first_flip})'
    print(msg)
    assert first_flip is None or first_flip >= 1, msg
    assert worst <= 1e-3, msg
    got = model([dev(im1), dev(im2)], training=False, flow_init=dev(fi))
    assert torch.equal(got[-1], ups[-1])


@pytest.mark.gpu
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('grid', [(9, 128), (13, 11)], ids=lambda g: f'{g[0]}x{g[1]}')
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_fused_loop_equals_the_public_ops_from_a_warm_state(T, variant, grid, precision):
    """raft_b200_forward_loop entered with coords1 = coords_init(flow_init), not the grid, gives byte for byte what the
    loop spelled out with CorrBlock.retrieve, update_block and upsample_flow gives from grid + flow_init, at every
    iteration and with last_only=True.  Batch 2."""
    h, w = grid
    iters, bs = 3, 2
    p = weights.init_params(variant, 1234, bias_scale=0.05, norm_jitter=0.1)
    im1, im2 = cases.images(bs, 8 * h, 8 * w, 3, 4)
    a, b = dev(im1), dev(im2)
    fi = dev(smooth_flow(bs, h, w, amp=4.0, seed=5))
    model = _model(T, variant, precision, p, iters)
    _, ups, _ = _spelled_out(T, model, a, b, fi, iters)
    full = model([a, b], training=False, flow_init=fi)
    assert len(full) == iters
    for i in range(iters):
        assert torch.equal(full[i], ups[i]), f'iteration {i}'
    last = model([a, b], training=False, last_only=True, flow_init=fi)
    assert len(last) == 1 and torch.equal(last[0], ups[-1])
    assert not torch.equal(model([a, b], training=False, last_only=True)[0], ups[-1]), 'flow_init was ignored'


@pytest.mark.gpu
def test_graph_replay_with_flow_init(T):
    """flow_init is a static input of the captured graph: replays with two different values each equal their eager call
    byte for byte (the buffer is re-read on every replay), and warm and cold calls of one shape never share a graph."""
    p = weights.init_params('raft', 7, bias_scale=0.02)
    eager = _model(T, 'raft', 'f16x2', p, 3)
    graph = _model(T, 'raft', 'f16x2', p, 3, use_graph=True)
    im1, im2 = cases.images(2, 64, 96, 40, 50)
    a, b = dev(im1), dev(im2)
    fa, fb = dev(smooth_flow(2, 8, 12, seed=1)), dev(smooth_flow(2, 8, 12, amp=5.0, seed=2))
    results = {}
    for name, fi in (('a', fa), ('b', fb), ('cold', None), ('a', fa), ('cold', None), ('b', fb)):
        want = eager([a, b], training=False, last_only=True, flow_init=fi)[-1].clone()
        got = graph([a, b], training=False, last_only=True, flow_init=fi)[-1].clone()
        assert torch.equal(got, want), name
        results[name] = got
    assert not torch.equal(results['a'], results['b'])
    assert not torch.equal(results['a'], results['cold'])
    assert len(graph._graphs) == 2


# --------------------------------------------------------------------------------------------- GPU: video
class _Counting:
    """Wraps an encoder and counts its calls and the images they encode."""

    def __init__(self, inner):
        self.inner, self.calls, self.images = inner, 0, 0

    def __call__(self, x, *args, **kwargs):
        self.calls += 1
        self.images += sum(t.shape[0] for t in x) if isinstance(x, (list, tuple)) else x.shape[0]
        return self.inner(x, *args, **kwargs)

    def __getattr__(self, name):
        return getattr(self.inner, name)


def _frames(bs, n, H, W, seed=90):
    return [dev(cases.images(bs, H, W, seed + t, seed + t)[0]) for t in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_predict_video_cold_equals_per_pair_calls(T, variant):
    """predict_video(warm_start=False) yields, for every t, exactly model([f_{t-1}, f_t], last_only=True)[-1], although
    it runs fnet T times on B images (each frame once) where per-pair calls encode 2B images per pair."""
    bs, n = 2, 5
    p = weights.init_params(variant, 1234, bias_scale=0.05, norm_jitter=0.1)
    model = _model(T, variant, 'f16x2', p, 3)
    frames = _frames(bs, n, 64, 96)
    want = [model([frames[t - 1], frames[t]], training=False, last_only=True)[-1].clone() for t in range(1, n)]
    model.fnet = _Counting(model.fnet)
    got = list(model.predict_video(iter(frames), warm_start=False))
    assert (model.fnet.calls, model.fnet.images) == (n, n * bs)
    assert len(got) == n - 1
    for t, (g, w) in enumerate(zip(got, want), start=1):
        assert tuple(g.shape) == (bs, 64, 96, 2)
        assert torch.equal(g, w), f'pair {t - 1} -> {t}'
    assert list(model.predict_video(frames[:1])) == [] and list(model.predict_video([])) == []
    with pytest.raises(ValueError):
        list(model.predict_video([frames[0], frames[1][:, :56]]))


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_predict_video_warm_equals_the_manual_chain(T, variant):
    """predict_video(warm_start=True) equals chaining __call__(flow_init=forward_interpolate(flow_low)) by hand, flow_low
    being coords1 - coords0 of the previous pair's last iteration; its first pair is the cold start."""
    bs, n = 2, 5
    p = weights.init_params(variant, 1234, bias_scale=0.05, norm_jitter=0.1)
    model = _model(T, variant, 'f16x2', p, 3)
    frames = _frames(bs, n, 64, 96, seed=120)
    got = list(model.predict_video(frames, warm_start=True))
    cold = list(model.predict_video(frames, warm_start=False))
    assert len(got) == n - 1 and torch.equal(got[0], cold[0])
    grid0 = T.coords_grid(bs, 8, 12)
    flow_init = None
    for t in range(1, n):
        want = model([frames[t - 1], frames[t]], training=False, last_only=True, flow_init=flow_init)[-1]
        assert torch.equal(got[t - 1], want), f'pair {t - 1} -> {t}'
        flow_init = T.forward_interpolate(model._last['coords1'] - grid0)
    assert not torch.equal(got[1], cold[1]), 'the warm start changed nothing'


@pytest.mark.gpu
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_predict_video_warm_vs_fp64_oracle(T, variant, precision):
    """Three frames through the fp64 oracle, with the NumPy forward interpolation between the pairs, against
    predict_video(warm_start=True): the 1e-3 max-abs gate on every iteration of every pair up to the first crossing of
    a discontinuity -- of the reference sampler (as in test_warm_start_vs_fp64_oracle) or of the forward interpolation
    (a target whose nearest source differs between the GPU's flow and the oracle's).  The per-iteration GPU values come
    from the loop spelled out with the public ops from the GPU's own warm start."""
    H, W, iters, n = 64, 128, 3, 3
    p = weights.init_params(variant, 77, bias_scale=0.02, norm_jitter=0.05)
    ims = [cases.images(1, H, W, 200 + t, 200 + t)[0] for t in range(n)]
    model = _model(T, variant, precision, p, iters)
    video = list(model.predict_video([dev(x) for x in ims], warm_start=True))
    assert len(video) == n - 1
    h, w = H // 8, W // 8
    grid_np = np.stack(np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64)), axis=-1)[None]
    fi_o = fi_g = None
    crossed = None
    for k in range(n - 1):
        want, inter = warm_start.forward(p, ims[k], ims[k + 1], variant, iters, dtype=torch.float64, flow_init=fi_o,
                                         return_intermediates=True)
        coords, ups, last = _spelled_out(T, model, dev(ims[k]), dev(ims[k + 1]), fi_g, iters)
        worst, first_flip = _gate(inter, want, coords, ups, model.corr_radius)
        print(f'{variant} {precision} pair {k}: max-abs {worst:.3e} before the first crossing (iteration {first_flip})')
        if crossed is None:
            assert worst <= 1e-3, f'pair {k}'
            if first_flip is not None:
                crossed = (k, first_flip)
            else:
                err = float((video[k].cpu().double() - want[-1]).abs().max())
                assert err <= 1e-3, f'pair {k}: predict_video max-abs {err:.3e}'
        flow_low_g = last - T.coords_grid(1, h, w)
        flow_low_o = (inter['coords'][-1].numpy() - grid_np).astype(F32)
        fi_g = T.forward_interpolate(flow_low_g)
        fi_o, idx_o = video_np.forward_interpolate(flow_low_o, return_index=True)
        fi_gn, idx_g = video_np.forward_interpolate(flow_low_g.cpu().numpy(), return_index=True)
        jump = (idx_g != idx_o) & (np.abs(fi_gn - fi_o).reshape(idx_o.shape + (2,)).max(-1) > 1e-3)
        if crossed is None and jump.any():
            crossed = (k + 1, 0)
    print(f'{variant} {precision}: first crossing (pair, iteration) = {crossed}')
    assert crossed is None or crossed >= (1, 1), 'the chain crossed a discontinuity before the first warm iteration'
