"""GPU: flow_to_image / flow_uv_to_colors (raft_b200_flow_to_image) byte for byte against the NumPy restatement
(oracle/flow_viz_np.py) outside the near-midpoint atan2 mask, from 1x1 to 1080x1920 and at radii from 1e-3 to 1e4, in
batches, at the edge cases of the reference's arithmetic, with a caller's rad_max, against the reference's own output
(tests/golden/flow_viz.npz), and through VisFlowCallback and predict_video.
"""
import os

import numpy as np
import pytest
import torch

from oracle import flow_viz_np as F
from test_flow_viz_ref import EXACT, GOLDEN, MAX_DIFFERING, _decode_png

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def V():
    from tf_raft_b200 import _lib, build
    import tf_raft_b200.datasets as D
    build.build()
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    return D


def _cmp(got, want, near, what):
    """Byte-equal outside the near-midpoint mask; inside it one level at most.  Returns the mask's size."""
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    assert got.shape == want.shape and got.dtype == np.uint8, (what, got.shape, want.shape)
    diff = (got != want).any(-1)
    if near.any():
        print(f'{what}: {int(near.sum())} near-midpoint pixels, {int((diff & near).sum())} of them differ')
    bad = diff & ~near
    assert not bad.any(), f'{what}: {int(bad.sum())} pixels differ, first {np.argwhere(bad)[:3].tolist()}: ' \
                          f'{got[bad][:3].tolist()} vs {want[bad][:3].tolist()}'
    assert np.abs(got.astype(int) - want.astype(int)).max(initial=0) <= 1, what
    return int(near.sum())


def _flow(rng, h, w, scale):
    return (rng.standard_normal((h, w, 2)) * scale).astype(np.float32)


@pytest.mark.parametrize('h,w', [(1, 1), (1, 37), (29, 1), (17, 31), (436, 1024), (448, 1024), (1080, 1920)])
def test_matches_restatement(V, h, w):
    """Byte-equal outside the near-midpoint mask.  The mask (|atan2 - midpoint| <= 2^-44 relative) holds about 2^-19 of
    random angles: 3, 2 and 10 pixels of the 4 x 436x1024, 4 x 448x1024 and 4 x 1080x1920 cases on an H100, where the
    one-level check above still applies."""
    rng = np.random.default_rng(h * 7919 + w)
    near_total = 0
    for scale in (1e-3, 1.0, 30.0, 1e4):
        flow = _flow(rng, h, w, scale)
        want, near = F.flow_to_image(flow)
        near_total += _cmp(V.flow_to_image(torch.from_numpy(flow).cuda()), want, near, f'{h}x{w} scale {scale}')
    print(f'{h}x{w}: {near_total} near-midpoint pixels')
    assert near_total <= 4 * h * w * 2.0 ** -17


def test_mixed_batch_equals_single_calls(V):
    rng = np.random.default_rng(16)
    flows = np.stack([_flow(rng, 37, 53, 10.0 ** rng.uniform(-3, 4)) for _ in range(16)])
    batch = V.flow_to_image(torch.from_numpy(flows).cuda()).cpu().numpy()
    for b in range(16):
        single = V.flow_to_image(torch.from_numpy(flows[b]).cuda()).cpu().numpy()
        assert np.array_equal(batch[b], single), b
        _cmp(batch[b], *F.flow_to_image(flows[b]), f'image {b}')


def test_edge_cases(V):
    def both(flow, **kw):
        want, near = F.flow_to_image(flow, **kw)
        got = V.flow_to_image(torch.from_numpy(flow).cuda(), **kw).cpu().numpy()
        assert not near.any()
        assert np.array_equal(got, want), (got, want)
        return got
    sz = both(np.array([[[5, 0], [5, -0.0], [-3, 0], [-3, -0.0], [0, 5], [-0.0, 5]]], np.float32))
    assert sz[0, 0].tolist() == [255, 0, 0] and sz[0, 1].tolist() == [255, 0, 43]
    assert (both(np.zeros((3, 4, 2), np.float32)) == 255).all()
    assert (both(np.array([[[2e19, 1], [1, 1], [-3e19, 0]]], np.float32)) == 255).all()       # rad_max = inf
    # the rad > 1 branch without a caller's rad_max: the largest pixel's normalised rad rounds to 1 + 2^-23
    flow = np.array([[[364.613525390625, 931.158935546875], [-8458.54, -5334.144], [0, -1]]], np.float32)
    for f in (flow[:, :1], flow[:, 1:]):
        d = np.max(np.sqrt(np.square(f[..., 0]) + np.square(f[..., 1]))) + np.float32(1e-5)
        assert F.steps(f[..., 0] / d, f[..., 1] / d)['rad'][0, 0] > 1
        both(f)
    # the clip: negatives, -0.0, +-inf and values above the bound
    flow = np.array([[[-1, 2], [-0.0, 7], [np.inf, -np.inf], [3, -0.0], [0.5, 1e30]]], np.float32)
    both(flow, clip_flow=3.0)
    both(flow, clip_flow=0.0)


def _sector_boundaries():
    """float32 (1, N) u, v on the circle of radius 0.5 next to each sector boundary fk = k, k = 0..54: per k, the
    points of the angle (2k/54 - 1) pi with u moved by up to 256 ulps whose restated fk is the largest below k and the
    smallest at or above k (fk = k itself where the float32 chain reaches it: always at k = 0 and 54).  Points with a
    near-midpoint atan2 are skipped.  Returns u, v and the number of exact integers reached."""
    us, vs, exact = [], [], 0
    for k in range(55):
        theta = (2 * k / 54 - 1) * np.pi
        u0, v0 = np.float32(-0.5 * np.cos(theta)), np.float32(-0.5 * np.sin(theta))
        cand = (np.array([u0] * 513, np.float32).view(np.int32) + np.arange(-256, 257, dtype=np.int32)).view(np.float32)
        s = F.steps(cand, np.full(513, v0, np.float32))
        fk = np.where(F.near_midpoint(s['a64']), np.nan, s['fk'])
        below, above = np.flatnonzero(fk < k), np.flatnonzero(fk >= k)
        picks = ([below[np.argmax(fk[below])]] if len(below) else []) + [above[np.argmin(fk[above])]]
        exact += int(fk[picks[-1]] == k)
        us += [cand[i] for i in picks]
        vs += [v0] * len(picks)
    return np.array([us], np.float32), np.array([vs], np.float32), exact


def test_sector_boundaries(V):
    """fk exactly each integer 0..54, k0 = 54 wrapping k1 to 0 included: flows planted by searching, per sector, for
    float32 (u, v) on a circle of radius 0.5 whose restated fk is that integer."""
    u, v, exact = _sector_boundaries()
    s = F.steps(u, v)
    assert set(s['k0'][0].tolist()) == set(range(55)) and s['fk'][0, 0] == 0 and s['fk'][0, -1] == 54
    assert s['k1'][0, -1] == 0 and exact >= 2
    want, near = F.flow_uv_to_colors(u, v)
    got = V.flow_uv_to_colors(torch.from_numpy(u).cuda(), torch.from_numpy(v).cuda())
    assert not near.any() and np.array_equal(got.cpu().numpy(), want)


def test_bgr_is_rgb_reversed(V):
    flow = torch.from_numpy(_flow(np.random.default_rng(2), 33, 47, 5.0)).cuda()
    rgb = V.flow_to_image(flow)
    assert torch.equal(V.flow_to_image(flow, convert_to_bgr=True), rgb.flip(-1))
    assert torch.equal(V.flow_to_image(flow, 2.0, True), V.flow_to_image(flow, 2.0).flip(-1))


def test_rad_max(V):
    rng = np.random.default_rng(5)
    flows = np.stack([_flow(rng, 31, 45, s) for s in (0.01, 1.0, 100.0)])
    t = torch.from_numpy(flows).cuda()
    own = np.array([np.max(np.sqrt(np.square(f[..., 0]) + np.square(f[..., 1]))) for f in flows], np.float32)
    assert torch.equal(V.flow_to_image(t, rad_max=torch.from_numpy(own).cuda()), V.flow_to_image(t))
    assert torch.equal(V.flow_to_image(t[1], rad_max=float(own[1])), V.flow_to_image(t[1]))
    got = V.flow_to_image(t, rad_max=1.5).cpu().numpy()                  # one scale for all three images
    darkened = 0
    for b in range(3):
        want, near = F.flow_to_image(flows[b], rad_max=1.5)
        _cmp(got[b], want, near, f'image {b}')
        darkened += int((np.sqrt(np.square(flows[b] / np.float32(1.5 + 1e-5)).sum(-1)) > 1).sum())
    assert darkened > 1000                                               # the 0.75 branch is exercised
    want, near = F.flow_to_image(flows[2], clip_flow=50.0, rad_max=0.0)
    _cmp(V.flow_to_image(t[2], 50.0, rad_max=0.0), want, near, 'rad_max 0 with clip')


def test_golden(V):
    g = np.load(GOLDEN)
    differing = 0
    for name, (flow, kw) in F.golden_cases().items():
        got = V.flow_to_image(torch.from_numpy(flow).cuda(), **kw).cpu().numpy()
        d = np.abs(got.astype(int) - g[name].astype(int))
        assert d.max() <= 1, name
        differing += int((d.max(-1) > 0).sum())
        if name in EXACT:
            assert np.array_equal(got, g[name]), name
    assert differing <= MAX_DIFFERING, differing


def test_errors(V):
    f = torch.zeros(4, 6, 7, 2, device='cuda')
    for k, val in ((2, float('nan')), (1, float('inf')), (3, -float('inf'))):
        g = f.clone()
        g[k, 3, 2, 1] = val
        with pytest.raises(ValueError, match=f'image {k} '):
            V.flow_to_image(g)
        with pytest.raises(ValueError, match=f'image {k} '):
            V.flow_to_image(g, rad_max=1.0)
    g = f.clone()
    g[1, 0, 0, 0], g[2, 1, 1, 1] = float('inf'), -float('inf')
    assert V.flow_to_image(g, clip_flow=4.0).shape == (4, 6, 7, 3)         # clipped to finite values
    g[3, 2, 2, 0] = float('nan')
    with pytest.raises(ValueError, match='image 3 '):
        V.flow_to_image(g, clip_flow=4.0)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        V.flow_to_image(f.cpu())
    for bad in (torch.zeros(6, 7, 3, device='cuda'), torch.zeros(6, 2, device='cuda'), torch.zeros(0, 7, 2, device='cuda'),
                torch.zeros(2, 6, 0, 2, device='cuda')):
        with pytest.raises(ValueError):
            V.flow_to_image(bad)
    for bad in (-1.0, float('inf'), float('nan'), 1e39):
        with pytest.raises(ValueError, match='rad_max'):
            V.flow_to_image(f, rad_max=bad)
        with pytest.raises(ValueError, match='clip_flow'):
            V.flow_to_image(f, clip_flow=bad)
    with pytest.raises(ValueError, match='rad_max of image 2'):
        V.flow_to_image(f, rad_max=torch.tensor([1.0, 2.0, -1.0, float('nan')], device='cuda'))
    with pytest.raises(ValueError, match='rad_max'):
        V.flow_to_image(f, rad_max=torch.ones(3, device='cuda'))
    with pytest.raises(ValueError):
        V.flow_uv_to_colors(torch.zeros(3, 4, device='cuda'), torch.zeros(4, 3, device='cuda'))


def test_flow_uv_to_colors(V):
    rng = np.random.default_rng(9)
    u = (rng.standard_normal((3, 19, 23)) * 0.7).astype(np.float32)
    v = (rng.standard_normal((3, 19, 23)) * 0.7).astype(np.float32)
    u[0, 0, 0], v[1, 2, 3], u[2, 4, 5], v[2, 4, 5] = np.inf, -np.inf, 1e30, -1e30
    got = V.flow_uv_to_colors(torch.from_numpy(u).cuda(), torch.from_numpy(v).cuda(), convert_to_bgr=True).cpu().numpy()
    for b in range(3):
        _cmp(got[b], *F.flow_uv_to_colors(u[b], v[b], True), f'image {b}')
    single = V.flow_uv_to_colors(torch.from_numpy(u[1]).cuda(), torch.from_numpy(v[1]).cuda(), True)
    assert np.array_equal(single.cpu().numpy(), got[1])
    v[1, 0, 0] = np.nan
    with pytest.raises(ValueError, match='image 1 '):
        V.flow_uv_to_colors(torch.from_numpy(u).cuda(), torch.from_numpy(v).cuda())


@pytest.mark.parametrize('choose_random', [False, True])
def test_vis_flow_callback(V, tmp_path, choose_random):
    import tf_raft_b200 as T
    rng = np.random.default_rng(11)
    data = [tuple(rng.integers(0, 256, (60, 90, 3), dtype=np.uint8) for _ in range(2)) + ('extra',) for _ in range(2)]
    model = T.RAFT(iters_pred=3, seed=0)
    cb = T.VisFlowCallback(data, target_size=(64, 96), num_visualize=1 if choose_random else 2,
                           choose_random=choose_random, logdir=str(tmp_path / 'vis'))
    cb.set_model(model)
    np.random.seed(4)
    cb.on_epoch_end(6)
    np.random.seed(4)
    ids = np.random.choice(2, size=1, replace=False) if choose_random else range(2)
    assert sorted(os.listdir(tmp_path / 'vis')) == [f'epoch007_{i + 1:03d}.png' for i in sorted(ids)]
    for i in ids:
        im1, im2, _ = data[i]
        pair = [T.resize_with_crop_or_pad(torch.from_numpy(im).float().cuda(), 64, 96)[None] for im in (im1, im2)]
        flow = T.resize_with_crop_or_pad(model(pair, training=False, last_only=True)[-1][0], 60, 90)
        want = np.concatenate([im1, im2, V.flow_to_image(flow).cpu().numpy()], axis=0)
        got = _decode_png((tmp_path / 'vis' / f'epoch007_{i + 1:03d}.png').read_bytes())
        assert np.array_equal(got, want), i
    with pytest.raises(ValueError, match='batched'):
        bad = T.VisFlowCallback([(np.zeros((1, 60, 90, 3)), np.zeros((1, 60, 90, 3)))], logdir=str(tmp_path / 'b'))
        bad.set_model(model)
        bad.on_epoch_end(0)


def test_predict_video_coloured_per_frame(V):
    import tf_raft_b200 as T
    rng = np.random.default_rng(12)
    frames = [torch.from_numpy(rng.uniform(0, 255, (2, 64, 96, 3)).astype(np.float32)).cuda() for _ in range(3)]
    model = T.RAFT(iters_pred=2, seed=1)
    for flow in model.predict_video(frames):
        batch = V.flow_to_image(flow, rad_max=20.0)
        for b in range(2):
            assert torch.equal(batch[b], V.flow_to_image(flow[b], rad_max=20.0))
            assert torch.equal(V.flow_to_image(flow)[b], V.flow_to_image(flow[b]))
