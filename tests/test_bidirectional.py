"""Bidirectional flow with forward-backward occlusion masks: `fb_occlusion`, `RAFT.predict_bidirectional` and
`predict_video(..., bidirectional=True)`.

CPU: the NumPy restatement of the consistency check (oracle.occlusion_np) against an fp64 formulation on
scipy.ndimage.map_coordinates and against analytic masks; host-side argument checks of raft_b200_fb_occlusion.  GPU: the
kernel bit for bit against NumPy; both directions run as one batch-2B loop equal the two single-direction calls; CUDA-graph
replay; the bidirectional video generator, cold and warm, against per-pair calls and the manual chain; the backward warm
start against the fp64 oracle.
"""
import ctypes

import numpy as np
import pytest
import torch

import cases
from oracle import occlusion_np, video_np, warm_start, weights
from test_video import _Counting, _frames, _gate, _model, _spelled_out, dev, smooth_flow

F32 = np.float32
ALPHAS = [(0.01, 0.5), (0.05, 1.25), (0.0, 0.0)]


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


# --------------------------------------------------------------------------------------------- CPU: the restatement
def fp64_occlusion(F, G, alpha1=0.01, alpha2=0.5):
    """An independent fp64 formulation of one direction: landing, closed-frame test, scipy's order-1 spline sample of G
    at the landing, the same threshold.  -> (occ, lhs, rhs), each (B, H, W)."""
    from scipy.ndimage import map_coordinates
    F, G = np.asarray(F, np.float64), np.asarray(G, np.float64)
    b, h, w, _ = F.shape
    gy, gx = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing='ij')
    occ = np.ones((b, h, w), bool)
    lhs, rhs = np.full((b, h, w), np.nan), np.full((b, h, w), np.nan)
    for k in range(b):
        px, py = gx + F[k, ..., 0], gy + F[k, ..., 1]
        inside = (px >= 0) & (px <= w - 1) & (py >= 0) & (py <= h - 1)
        at = np.stack([py[inside], px[inside]])
        g = np.stack([map_coordinates(G[k, ..., c], at, order=1, mode='nearest') for c in range(2)], axis=-1)
        f = F[k][inside]
        l = ((f + g) ** 2).sum(-1)
        r = alpha1 * ((f ** 2).sum(-1) + (g ** 2).sum(-1)) + alpha2
        lhs[k][inside], rhs[k][inside] = l, r
        occ[k][inside] = ~(l <= r)
    return occ, lhs, rhs


def translation(b, h, w, t):
    """F = t everywhere, G = -t everywhere: every landing inside the frame is consistent."""
    F = np.broadcast_to(np.asarray(t, F32), (b, h, w, 2)).copy()
    return F, -F


def _strip(h, w, t):
    """Pixels whose landing (x + tx, y + ty) leaves the closed frame."""
    gy, gx = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing='ij')
    px, py = gx + t[0], gy + t[1]
    return ~((px >= 0) & (px <= w - 1) & (py >= 0) & (py <= h - 1))


@pytest.mark.parametrize('kind', ['smooth', 'translation', 'corrupted'])
def test_numpy_fb_occlusion_matches_fp64(kind):
    """oracle.occlusion_np equals the fp64 formulation wherever |lhs - rhs| is not within 1e-5 relative of the threshold
    (no texel is non-finite here).  Exact inverse translations are consistent everywhere except the strip whose landing
    leaves the frame; a corrupted rectangle in G flags exactly the forward pixels whose bilinear support touches it and,
    backward, exactly the rectangle (plus the strip)."""
    b, h, w = 2, 23, 31
    t = (2.5, -1.25)
    if kind == 'smooth':
        F = smooth_flow(b, h, w, amp=3.0, seed=4)
        G = -smooth_flow(b, h, w, amp=3.0, seed=4) + np.random.default_rng(5).normal(0, 0.4, (b, h, w, 2)).astype(F32)
    else:
        F, G = translation(b, h, w, t)
        if kind == 'corrupted':
            G[:, 5:11, 7:19] += F32([20.0, -15.0])
    want = occlusion_np.fb_occlusion(F, G, return_terms=True)
    assert want[0][0].dtype == bool and want[0][0].shape == (b, h, w)
    for (occ, inside, lhs, rhs), (A, Bf) in zip(want, ((F, G), (G, F))):
        occ64, lhs64, rhs64 = fp64_occlusion(A, Bf)
        near = np.abs(lhs64 - rhs64) <= 1e-5 * np.abs(rhs64)
        agree = (occ == occ64) | near
        assert agree.all(), f'{int((~agree).sum())} pixels differ from the fp64 formulation'
        assert (inside == ~np.isnan(lhs64)).all()
    if kind == 'smooth':
        for occ, *_ in want:
            assert 0 < occ.mean() < 0.9
        return
    occ_fw, occ_bw = want[0][0], want[1][0]
    strip_fw, strip_bw = _strip(h, w, t), _strip(h, w, (-t[0], -t[1]))
    assert strip_fw.any() and not strip_fw.all()
    if kind == 'translation':
        np.testing.assert_array_equal(occ_fw, np.broadcast_to(strip_fw, occ_fw.shape))
        np.testing.assert_array_equal(occ_bw, np.broadcast_to(strip_bw, occ_bw.shape))
        return
    rect = np.zeros((h, w), bool)
    rect[5:11, 7:19] = True
    gy, gx = np.meshgrid(np.arange(h), np.arange(w), indexing='ij')
    x0, y0 = np.floor(gx + t[0]).astype(int), np.floor(gy + t[1]).astype(int)
    touch = np.zeros((h, w), bool)                    # ax = 0.5, ay = 0.75 at every landing: all four texels weigh
    for dy in (0, 1):
        for dx in (0, 1):
            yy, xx = np.clip(y0 + dy, 0, h - 1), np.clip(x0 + dx, 0, w - 1)
            touch |= rect[yy, xx]
    np.testing.assert_array_equal(occ_fw, np.broadcast_to(strip_fw | touch, occ_fw.shape))
    np.testing.assert_array_equal(occ_bw, np.broadcast_to(strip_bw | rect, occ_bw.shape))


def test_host_side_argument_errors_of_fb_occlusion(L):
    """raft_b200_fb_occlusion validates on the host like the other entry points: NULL pointers, negative, NaN or
    infinite thresholds and flows not 8-byte aligned (float2 loads) -> RAFT_ERR_BAD_ARG; non-positive B, H or W ->
    RAFT_ERR_BAD_SHAPE."""
    fake, odd = ctypes.c_void_p(0x1000), ctypes.c_void_p(0x1004)
    fn = L.raft_b200_fb_occlusion
    for i in range(4):
        ptrs = [fake] * 4
        ptrs[i] = None
        assert fn(ptrs[0], ptrs[1], 1, 8, 8, 0.01, 0.5, ptrs[2], ptrs[3], None) == -1
    for bad in (-1.0, -1e-30, float('nan'), float('inf')):
        assert fn(fake, fake, 1, 8, 8, bad, 0.5, fake, fake, None) == -1
        assert fn(fake, fake, 1, 8, 8, 0.01, bad, fake, fake, None) == -1
    assert fn(odd, fake, 1, 8, 8, 0.01, 0.5, fake, fake, None) == -1
    assert fn(fake, odd, 1, 8, 8, 0.01, 0.5, fake, fake, None) == -1
    for B, H, W in ((0, 8, 8), (1, -3, 8), (1, 8, 0), (-1, 1, 1)):
        assert fn(fake, fake, B, H, W, 0.01, 0.5, fake, fake, None) == -2
    assert L.raft_b200_abi_version() == 2


# --------------------------------------------------------------------------------------------- GPU: the kernel
def _equality_flow(alpha1, alpha2):
    """Float32 (v, u), v, u >= 0, with v*v + u*u == alpha1*((v*v + u*u) + (0*0 + 0*0)) + alpha2 exactly in float32: the
    flow (v, u) against zero backward flow sits exactly on the threshold.  For a fixed u, lhs - rhs crosses zero once as
    v steps through the floats, and a step of v moves v*v by about two ulps, so several u are tried."""
    a1, a2, z = F32(alpha1), F32(alpha2), F32(0)
    for u in np.arange(0, 1, 1 / 16, dtype=F32):
        root = np.sqrt(max(np.float64(alpha2) / (1.0 - np.float64(alpha1)) - np.float64(u) ** 2, 0.0)).astype(F32)
        v = np.abs((root.view(np.int32) + np.arange(-4000, 4000, dtype=np.int32)).view(F32))
        lhs = v * v + u * u
        rhs = a1 * ((v * v + u * u) + (z * z + z * z)) + a2
        hit = v[lhs == rhs]
        if hit.size:
            return hit[np.argmin(np.abs(hit - root))], u
    raise AssertionError('no exact equality found')


def occ_case(b, h, w, alpha1, alpha2, seed):
    """(F, G, planted) for batch b >= 3: image 0 a smooth flow against a noisy inverse, with NaN and +-inf in F and G;
    image 1 zero G with pixels planted exactly on the threshold; image 2 exact and one-ulp-outside landings on both
    frame edges, integer landings reading a NaN texel at weight 0.  `planted` maps a name to its (b, y, x) indices."""
    rng = np.random.default_rng(seed)
    F = smooth_flow(b, h, w, amp=min(3.0, max(h, w) / 4), seed=seed)
    G = -F + rng.normal(0, 0.3, F.shape).astype(F32)
    planted = {}
    n = h * w
    k = max(1, n // 40)

    def pick(img, m):
        sel = rng.choice(n, size=min(n, m), replace=False)
        return np.full(sel.size, img), sel // w, sel % w

    for arr, c, val in ((F, 0, np.nan), (F, 1, np.inf), (G, 0, -np.inf), (G, 1, np.nan)):
        i, y, x = pick(0, k)
        arr[i, y, x, c] = val
    # image 1: G = 0, F = (+-v, u) lands inside -> lhs == rhs exactly
    G[1] = 0
    v, u = _equality_flow(alpha1, alpha2)
    i, y, x = pick(1, 3 * k)
    ok = (x + v <= w - 1) & (y + u <= h - 1)
    F[i[ok], y[ok], x[ok]] = (v, u)
    okm = ~ok & (x - v >= 0) & (y + u <= h - 1)
    F[i[okm], y[okm], x[okm]] = (-v, u)
    planted['threshold'] = (i[ok | okm], y[ok | okm], x[ok | okm])
    # image 2, disjoint pixel sets: landings exactly on 0 / W-1 / H-1, and one float32 ulp outside (x + fx exact)
    perm = rng.permutation(n)
    chunks = iter(np.array_split(perm[:9 * k], 9)) if n >= 9 * k else iter([perm[j:j + 1] for j in range(9)])

    def take():
        sel = next(chunks)
        return np.full(sel.size, 2), sel // w, sel % w

    gx = np.arange(w, dtype=F32)[None, :]
    gy = np.arange(h, dtype=F32)[:, None]
    inf = F32(np.inf)
    edge = {'x=0': (0, -gx), 'x=W-1': (0, F32(w - 1) - gx), 'y=0': (1, -gy), 'y=H-1': (1, F32(h - 1) - gy)}
    out = {'x=0': (0, np.nextafter(-gx, -inf)), 'x=W-1': (0, np.nextafter(F32(w - 1), inf) - gx),
           'y=0': (1, np.nextafter(-gy, -inf)), 'y=H-1': (1, np.nextafter(F32(h - 1), inf) - gy)}
    for name, table in (('edge', edge), ('ulp_out', out)):
        for side, (c, val) in table.items():
            i, y, x = take()
            F[i, y, x] = 0                                     # the other component lands on the pixel itself
            F[i, y, x, c] = np.broadcast_to(val, (h, w))[y, x]
            planted[f'{name} {side}'] = (i, y, x)
    # integer landings: the texel right of the landing weighs 0 and holds NaN
    i, y, x = take()
    ix = rng.integers(0, w, x.size)
    iy = rng.integers(0, h, y.size)
    F[i, y, x] = np.stack([ix - x, iy - y], -1).astype(F32)
    G[i, iy, np.minimum(ix + 1, w - 1), 0] = np.nan
    planted['integer'] = (i, y, x)
    return F, G, planted


OCC_GRIDS = [(1, 1), (7, 5), (13, 11), (56, 64), (448, 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize('alphas', ALPHAS, ids=lambda a: f'a1={a[0]}_a2={a[1]}')
@pytest.mark.parametrize('grid', OCC_GRIDS, ids=lambda g: f'{g[0]}x{g[1]}')
def test_fb_occlusion_bit_exact(T, grid, alphas):
    """Both masks equal NumPy's float32 restatement exactly, batch 3: smooth flow against a noisy inverse, NaN and +-inf
    in F and G, pixels exactly on the threshold (consistent), landings exactly on the frame's edges (inside) and one ulp
    beyond them (occluded), integer landings whose zero-weight texel is NaN (occluded)."""
    h, w = grid
    a1, a2 = alphas
    F, G, planted = occ_case(3, h, w, a1, a2, seed=10 * h + w)
    (occ_fw, inside, lhs, rhs), want_bw = occlusion_np.fb_occlusion(F, G, a1, a2, return_terms=True)
    got_fw, got_bw = T.fb_occlusion(dev(F), dev(G), a1, a2)
    assert got_fw.dtype == torch.bool and tuple(got_fw.shape) == (3, h, w) and got_fw.device == dev(F).device
    np.testing.assert_array_equal(got_fw.cpu().numpy(), occ_fw)
    np.testing.assert_array_equal(got_bw.cpu().numpy(), want_bw[0])
    # the planted cases landed where intended (in the restatement the kernel equals)
    th = planted['threshold']
    if th[0].size:
        assert (lhs[th] == rhs[th]).all() and not occ_fw[th].any()
    for side in ('x=0', 'x=W-1', 'y=0', 'y=H-1'):
        assert inside[planted[f'edge {side}']].all(), side
        assert not inside[planted[f'ulp_out {side}']].any() and occ_fw[planted[f'ulp_out {side}']].all(), side
    assert occ_fw[planted['integer']].all()
    # defaults, and an unaligned view (copied before the float2 loads)
    np.testing.assert_array_equal(T.fb_occlusion(dev(F), dev(G))[1].cpu().numpy(),
                                  occlusion_np.fb_occlusion(F, G)[1])
    flat = torch.zeros(F.size + 1, device='cuda')
    flat[1:] = dev(F).reshape(-1)
    odd = flat[1:].view(F.shape)
    assert odd.data_ptr() % 8
    np.testing.assert_array_equal(T.fb_occlusion(odd, dev(G), a1, a2)[0].cpu().numpy(), occ_fw)


@pytest.mark.gpu
def test_fb_occlusion_argument_errors(T):
    F = dev(np.zeros((2, 8, 12, 2), F32))
    for a, b in ((F, F[:1]), (F, F[..., :1]), (F[..., :1], F[..., :1]), (F[0], F[0]), (F, F[:, :, :11])):
        with pytest.raises(ValueError):
            T.fb_occlusion(a, b)
    for a1, a2 in ((-0.01, 0.5), (0.01, -1.0), (float('nan'), 0.5), (0.01, float('inf')), (1e39, 0.5)):
        with pytest.raises(ValueError):
            T.fb_occlusion(F, F, a1, a2)
    with pytest.raises(TypeError):
        T.fb_occlusion(np.zeros((2, 8, 12, 2), F32), F)
    with pytest.raises(TypeError):
        T.fb_occlusion(F, torch.zeros((2, 8, 12, 2), dtype=torch.int32, device='cuda'))
    with pytest.raises(TypeError):
        T.fb_occlusion(F, F, 'a')
    with pytest.raises(RuntimeError):
        T.fb_occlusion(F, F.cpu())


# --------------------------------------------------------------------------------------------- GPU: predict_bidirectional
CONFIGS = [('f16x2', None), ('fp32', 'native')]


@pytest.mark.gpu
@pytest.mark.parametrize('precision,encoders', CONFIGS, ids=['f16x2', 'fp32-native'])
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_predict_bidirectional_equals_single_direction_calls(T, variant, precision, encoders):
    """Both directions as one batch-2B loop give exactly model([a, b]) and model([b, a]) (last_only, the final
    prediction), and the masks are fb_occlusion of those flows; fnet and cnet each run once on the 2B images."""
    bs = 2
    p = weights.init_params(variant, 1234, bias_scale=0.05, norm_jitter=0.1)
    model = _model(T, variant, precision, p, 3, encoder_backend=encoders)
    im1, im2 = cases.images(bs, 64, 96, 21, 22)
    a, b = dev(im1), dev(im2)
    model.fnet, model.cnet = _Counting(model.fnet), _Counting(model.cnet)
    got = [t.clone() for t in model.predict_bidirectional([a, b])]
    assert (model.fnet.calls, model.fnet.images) == (1, 2 * bs)
    assert (model.cnet.calls, model.cnet.images) == (1, 2 * bs)
    assert tuple(model._last['coords1'].shape) == (2 * bs, 8, 12, 2)
    flow_fw, flow_bw, occ_fw, occ_bw = got
    assert tuple(flow_fw.shape) == (bs, 64, 96, 2) and occ_fw.dtype == torch.bool and tuple(occ_bw.shape) == (bs, 64, 96)
    want_fw = model([a, b], training=False, last_only=True)[-1]
    want_bw = model([b, a], training=False, last_only=True)[-1]
    assert torch.equal(flow_fw, want_fw) and torch.equal(flow_bw, want_bw)
    want_occ = T.fb_occlusion(want_fw, want_bw)
    assert torch.equal(occ_fw, want_occ[0]) and torch.equal(occ_bw, want_occ[1])
    assert not torch.equal(flow_fw, -flow_bw)
    with pytest.raises(ValueError):
        model.predict_bidirectional([a, b[:, :56]])


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_predict_bidirectional_fp32_cudnn_vs_fp64_oracle(T, variant):
    """The default fp32 configuration (cuDNN encoders, whose algorithm may depend on the batch): each direction within
    1e-3 max-abs of the fp64 oracle of that direction at every iteration, up to the first crossing of a discontinuity
    of the reference sampler.  The per-iteration values are predict_bidirectional itself run for 1, 2, 3 iterations."""
    bs, H, W, iters = 2, 64, 96, 3
    p = weights.init_params(variant, 77, bias_scale=0.02, norm_jitter=0.05)
    im1, im2 = cases.images(bs, H, W, 11, 12)
    model = _model(T, variant, 'fp32', p, iters)
    assert model._encoder_backend() == 'torch'
    grid = T.coords_grid(2 * bs, H // 8, W // 8)
    ups, coords = [[], []], [[grid[:bs]], [grid[bs:]]]
    for k in range(1, iters + 1):
        model.iters_pred = k
        out = model.predict_bidirectional([dev(im1), dev(im2)])
        for d in range(2):
            ups[d].append(out[d].clone())
            coords[d].append(model._last['coords1'][d * bs:(d + 1) * bs].clone())
    for d, (x, y) in enumerate(((im1, im2), (im2, im1))):
        want, inter = warm_start.forward(p, x, y, variant, iters, dtype=torch.float64, return_intermediates=True)
        worst, first_flip = _gate(inter, want, coords[d][:iters], ups[d], model.corr_radius)
        msg = f'{variant} {"fw" if d == 0 else "bw"}: max-abs {worst:.3e} before the first crossing ({first_flip})'
        print(msg)
        assert first_flip is None or first_flip >= 1, msg
        assert worst <= 1e-3, msg


@pytest.mark.gpu
def test_predict_bidirectional_graph_replay(T):
    """use_graph=True: replays on two input pairs, alternately, equal the eager result byte for byte (flows and masks),
    and the bidirectional graph is kept apart from __call__'s graph at the same shape."""
    p = weights.init_params('raft', 7, bias_scale=0.02)
    eager = _model(T, 'raft', 'f16x2', p, 3)
    graph = _model(T, 'raft', 'f16x2', p, 3, use_graph=True)
    pairs = {'P': [dev(x) for x in cases.images(2, 64, 96, 40, 50)], 'Q': [dev(x) for x in cases.images(2, 64, 96, 60, 70)]}
    results = {}
    for name in ('P', 'Q', 'P', 'call', 'Q', 'P'):
        if name == 'call':
            want = eager(pairs['P'], training=False, last_only=True)[-1].clone()
            assert torch.equal(graph(pairs['P'], training=False, last_only=True)[-1], want)
            continue
        want = [t.clone() for t in eager.predict_bidirectional(pairs[name])]
        got = [t.clone() for t in graph.predict_bidirectional(pairs[name])]
        for i, (g, w) in enumerate(zip(got, want)):
            assert torch.equal(g, w), f'{name} output {i}'
        results[name] = got
    assert not torch.equal(results['P'][0], results['Q'][0])
    assert len(graph._graphs) == 2
    assert any(k[0] == 'bidirectional' for k in graph._graphs)


# --------------------------------------------------------------------------------------------- GPU: video
def _equal_tuples(got, want, what):
    assert len(got) == len(want) == 4
    for i, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w), f'{what}: output {i}'


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_bidirectional_video_cold_equals_predict_bidirectional(T, variant):
    """predict_video(bidirectional=True, warm_start=False) yields for every pair exactly predict_bidirectional of that
    pair, while fnet and cnet each run once per frame on B images."""
    bs, n = 2, 5
    p = weights.init_params(variant, 1234, bias_scale=0.05, norm_jitter=0.1)
    model = _model(T, variant, 'f16x2', p, 3)
    frames = _frames(bs, n, 64, 96, seed=150)
    want = [[x.clone() for x in model.predict_bidirectional([frames[t - 1], frames[t]])] for t in range(1, n)]
    model.fnet, model.cnet = _Counting(model.fnet), _Counting(model.cnet)
    got = list(model.predict_video(iter(frames), warm_start=False, bidirectional=True))
    assert (model.fnet.calls, model.fnet.images) == (model.cnet.calls, model.cnet.images) == (n, n * bs)
    assert len(got) == n - 1
    for t, (g, w) in enumerate(zip(got, want), start=1):
        _equal_tuples(g, w, f'pair {t - 1} -> {t}')
    assert list(model.predict_video(frames[:1], bidirectional=True)) == []
    assert list(model.predict_video([], bidirectional=True)) == []


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_bidirectional_video_warm_equals_the_manual_chain(T, variant):
    """predict_video(bidirectional=True, warm_start=True): the forward half chains __call__ with
    flow_init=forward_interpolate(F_low), the backward half __call__ on the reversed pair with
    flow_init=-forward_interpolate(-B_low), bit for bit; its forward flows are those of bidirectional=False; and the
    warm start changes the backward flow of the second pair."""
    bs, n = 2, 4
    p = weights.init_params(variant, 1234, bias_scale=0.05, norm_jitter=0.1)
    model = _model(T, variant, 'f16x2', p, 3)
    frames = _frames(bs, n, 64, 96, seed=170)
    got = list(model.predict_video(frames, warm_start=True, bidirectional=True))
    cold = list(model.predict_video(frames, warm_start=False, bidirectional=True))
    uni = list(model.predict_video(frames, warm_start=True))
    assert len(got) == len(uni) == n - 1
    _equal_tuples(got[0], cold[0], 'first pair')
    grid0 = T.coords_grid(bs, 8, 12)
    fi_f = fi_b = None
    for t in range(1, n):
        fw = model([frames[t - 1], frames[t]], training=False, last_only=True, flow_init=fi_f)[-1].clone()
        f_low = model._last['coords1'] - grid0
        bw = model([frames[t], frames[t - 1]], training=False, last_only=True, flow_init=fi_b)[-1].clone()
        b_low = model._last['coords1'] - grid0
        _equal_tuples(got[t - 1], (fw, bw) + T.fb_occlusion(fw, bw), f'pair {t - 1} -> {t}')
        assert torch.equal(got[t - 1][0], uni[t - 1]), f'forward flow of pair {t - 1} -> {t}'
        fi_f, fi_b = T.forward_interpolate(f_low), -T.forward_interpolate(-b_low)
    assert not torch.equal(got[1][1], cold[1][1]), 'the backward warm start changed nothing'


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['f16x2', 'fp32'])
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_backward_warm_start_vs_fp64_oracle(T, variant, precision):
    """Three frames through the fp64 oracle on the reversed pairs, with the NumPy -forward_interpolate(-B_low) between
    them, against the backward flows of predict_video(bidirectional=True, warm_start=True): the 1e-3 max-abs gate on
    every iteration up to the first crossing of a discontinuity, counted as in
    test_video.test_predict_video_warm_vs_fp64_oracle (the reference sampler, or a target whose forward-interpolation
    source differs between the GPU's flow and the oracle's).  The per-iteration GPU values come from the loop spelled
    out with the public ops from the GPU's own backward warm start."""
    H, W, iters, n = 64, 128, 3, 3
    p = weights.init_params(variant, 77, bias_scale=0.02, norm_jitter=0.05)
    ims = [cases.images(1, H, W, 200 + t, 200 + t)[0] for t in range(n)]
    model = _model(T, variant, precision, p, iters)
    video = list(model.predict_video([dev(x) for x in ims], warm_start=True, bidirectional=True))
    assert len(video) == n - 1
    h, w = H // 8, W // 8
    grid_np = np.stack(np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64)), axis=-1)[None]
    fi_o = fi_g = None
    crossed = None
    for k in range(n - 1):
        want, inter = warm_start.forward(p, ims[k + 1], ims[k], variant, iters, dtype=torch.float64, flow_init=fi_o,
                                         return_intermediates=True)
        coords, ups, last = _spelled_out(T, model, dev(ims[k + 1]), dev(ims[k]), fi_g, iters)
        worst, first_flip = _gate(inter, want, coords, ups, model.corr_radius)
        print(f'{variant} {precision} pair {k}: max-abs {worst:.3e} before the first crossing (iteration {first_flip})')
        if crossed is None:
            assert worst <= 1e-3, f'pair {k}'
            if first_flip is not None:
                crossed = (k, first_flip)
            else:
                err = float((video[k][1].cpu().double() - want[-1]).abs().max())
                assert err <= 1e-3, f'pair {k}: backward flow max-abs {err:.3e}'
        neg_low_g = -(last - T.coords_grid(1, h, w))
        neg_low_o = -(inter['coords'][-1].numpy() - grid_np).astype(F32)
        fi_g = -T.forward_interpolate(neg_low_g)
        fo, idx_o = video_np.forward_interpolate(neg_low_o, return_index=True)
        fi_o = -fo
        fg, idx_g = video_np.forward_interpolate(neg_low_g.cpu().numpy(), return_index=True)
        jump = (idx_g != idx_o) & (np.abs(fg - fo).reshape(idx_o.shape + (2,)).max(-1) > 1e-3)
        if crossed is None and jump.any():
            crossed = (k + 1, 0)
    print(f'{variant} {precision}: first crossing (pair, iteration) = {crossed}')
    assert crossed is None or crossed >= (1, 1), 'the chain crossed a discontinuity before the first warm iteration'
