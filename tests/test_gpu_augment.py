"""GPU: FlowAugmentor / SparseFlowAugmentor (raft_b200_augment_dense / _sparse) bit for bit against the NumPy restatement
(oracle/augment_np.py): images, flow and valid, over every branch of the reference's augmentors, at Chairs, Sintel and
KITTI sizes, in mixed-size batches, with planted flows at the valid threshold and non-finite flows, and dense KITTI
collisions; then one train_step on an augmented batch.
"""
import random

import numpy as np
import pytest
import torch

from oracle import augment_np as A

pytestmark = pytest.mark.gpu

CHAIRS, SINTEL, KITTI = (384, 512), (436, 1024), (375, 1242)
CROP_DENSE, CROP_SINTEL, CROP_KITTI = (368, 496), (368, 768), (288, 960)


@pytest.fixture(scope='module')
def M():
    from tf_raft_b200 import _lib, build
    import tf_raft_b200.datasets as D
    build.build()
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    return D


def _sample(rng, h, w, sparse=False, density=0.3):
    img1 = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    img2 = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    # smooth-ish images so that the HSV round trip meets grey, saturated and every sector
    img1[: h // 4] = img1[: h // 4, :1]
    flow = (rng.standard_normal((h, w, 2)) * 20).astype(np.float32)
    if not sparse:
        return img1, img2, flow
    valid = (rng.uniform(size=(h, w)) < density).astype(np.float32)
    return img1, img2, flow, valid


def _bits(x):
    x = np.ascontiguousarray(x, dtype=np.float32).copy()
    x[np.isnan(x)] = np.nan                                   # one NaN pattern: NumPy and the GPU differ in its sign
    return x.view(np.uint32)


def _check(aug, samples, params, sparse):
    got = [t.cpu().numpy() for t in aug.batch([tuple(torch.from_numpy(a).cuda() for a in s) for s in samples], params)]
    for i, (s, p) in enumerate(zip(samples, params)):
        want = A.augment_sparse(*s, p) if sparse else A.augment_dense(*s, p)
        for k, name in enumerate(('img1', 'img2', 'flow', 'valid')):
            g, w = got[k][i], want[k]
            ok = np.array_equal(g, w) if k < 2 else np.array_equal(_bits(g), _bits(w))
            if not ok:
                bad = np.argwhere((g != w) if k < 2 else (_bits(g) != _bits(w)))
                raise AssertionError(f'sample {i} {name}: {len(bad)} differ, first {bad[:3].tolist()}: '
                                     f'{g[tuple(bad[0])]} vs {w[tuple(bad[0])]}; params {p}')
    return got


def _P(D, crop, colour1=(None, None), colour2=None, rects=(), sx=1.0, sy=None, spatial=False, hflip=False, vflip=False,
       y0=0, x0=0):
    return D.AugmentParams(colour1, colour1 if colour2 is None else colour2, list(rects), sx, sx if sy is None else sy,
                           spatial, hflip, vflip, y0, x0, crop)


BC, HSV = (1.23, -0.17), (-21.7, 88.4, 0.0)


def test_branches_chairs(M):
    """Hand-picked parameter sets over Chairs sources: spatial on/off, stretch, each flip, symmetric and asymmetric
    colour with each gate on/off, 0/1/2 eraser rectangles including ones crossing the right and bottom borders."""
    rng = np.random.default_rng(1)
    crop = CROP_DENSE
    h, w = CHAIRS
    s = 1.0527
    ps = [
        _P(M, crop),
        _P(M, crop, colour1=(BC, None), sx=s, spatial=True, y0=30, x0=20),
        _P(M, crop, colour1=(None, HSV), sx=s, sy=s * 1.11, spatial=True, hflip=True, y0=9, x0=41),
        _P(M, crop, colour1=(BC, HSV), colour2=(None, (5.5, -40.2, 0.0)), rects=[(500, 370, 77, 60)], vflip=True,
           y0=16, x0=16),
        _P(M, crop, colour1=((0.7, 0.35), HSV), colour2=((1.31, -0.05), None),
           rects=[(3, 4, 99, 51), (480, 10, 80, 99)], sx=1.4, sy=0.99, spatial=True, hflip=True, vflip=True, y0=12,
           x0=200),
        _P(M, crop, colour1=(None, (27.9, 101.9, 0.0)), rects=[(0, 0, 50, 50)], sx=0.9767, spatial=True, y0=7, x0=4),
    ]
    samples = [_sample(rng, h, w) for _ in ps]
    _check(M.FlowAugmentor(crop), samples, ps, False)


def test_hsv_row_tail_at_kitti_widths(M):
    """HSV round trips at widths 1242 and 1226, whose last W mod 32 columns take cv2's rounding row tail, dense and
    sparse, with and without the resize."""
    rng = np.random.default_rng(2)
    for cls, sparse in ((M.FlowAugmentor, False), (M.SparseFlowAugmentor, True)):
        shapes = [KITTI, (370, 1226)]
        samples = [_sample(rng, *s, sparse=sparse) for s in shapes for _ in range(2)]
        ps = [_P(M, CROP_KITTI, colour1=(None, HSV), colour2=(BC, (11.3, -60.1, 0.0)) if not sparse else None),
              _P(M, CROP_KITTI, colour1=(BC, HSV), sx=0.8317, spatial=True, y0=5, x0=30),
              _P(M, CROP_KITTI, colour1=((0.8, 0.1), (-27.5, 33.3, 0.0)), y0=60, x0=200),
              _P(M, CROP_KITTI, colour1=(None, (3.9, 101.2, 0.0)), sx=0.97, spatial=True, hflip=True, y0=11, x0=17)]
        _check(cls(CROP_KITTI), samples, ps, sparse)


@pytest.mark.parametrize('kind,shape,crop', [('dense', CHAIRS, CROP_DENSE), ('dense', SINTEL, CROP_SINTEL),
                                             ('sparse', KITTI, CROP_KITTI)])
def test_seeded_samples(M, kind, shape, crop):
    """Parameters from the seeded sampler, 12 samples in batches of 4, at the dataset's size."""
    rng = np.random.default_rng(5)
    aug = (M.FlowAugmentor if kind == 'dense' else M.SparseFlowAugmentor)(crop, do_flip=True)
    np.random.seed(3)
    random.seed(4)
    for _ in range(3):
        samples = [_sample(rng, *shape, sparse=kind == 'sparse') for _ in range(4)]
        params = [aug.sample_params(*shape) for _ in samples]
        _check(aug, samples, params, kind == 'sparse')


def test_mixed_sizes_one_launch(M):
    """Chairs, Sintel and an odd size in one dense launch equal the per-sample calls (and the oracle)."""
    rng = np.random.default_rng(8)
    aug = M.FlowAugmentor(CROP_DENSE)
    np.random.seed(21)
    random.seed(22)
    shapes = [CHAIRS, SINTEL, (401, 611), CHAIRS, SINTEL]
    samples = [_sample(rng, *s) for s in shapes]
    params = [aug.sample_params(*s) for s in shapes]
    got = _check(aug, samples, params, False)
    for i, (s, p) in enumerate(zip(samples, params)):
        one = aug(*(torch.from_numpy(a).cuda() for a in s), params=p)
        for k in range(3):
            assert torch.equal(one[k].cpu(), torch.from_numpy(got[k][i])), (i, k)


def test_identity_is_a_crop(M):
    rng = np.random.default_rng(9)
    s = _sample(rng, *CHAIRS)
    img1, img2, flow = M.FlowAugmentor(CROP_DENSE)(*(torch.from_numpy(a).cuda() for a in s),
                                                   params=_P(M, CROP_DENSE, y0=5, x0=11))
    sl = np.s_[5:5 + CROP_DENSE[0], 11:11 + CROP_DENSE[1]]
    assert np.array_equal(img1.cpu().numpy(), s[0][sl]) and np.array_equal(img2.cpu().numpy(), s[1][sl])
    assert np.array_equal(flow.cpu().numpy().view(np.uint32), s[2][sl].view(np.uint32))


def test_valid_threshold_and_nonfinite_flow(M):
    """Flows whose fp64 value is below 1000 but whose float32 cast is 1000 stay valid, as dataset.py:102 decides on the
    fp64 flow; NaN and +-inf source flow, resized and copied."""
    h, w = CHAIRS
    crop = CROP_DENSE

    def planted(f, v):
        return (v == 1) & ((np.abs(f[..., 0]) == 1000) | (np.abs(f[..., 1]) == 1000))

    # flow within 40 float32 ulps of 1000 / scale; whether a product lands in [1000 - ulp/2, 1000) depends on the
    # scale's bits, so the first scale whose oracle output has such pixels is used
    for sx in (1.0371, 1.0437, 1.0519, 1.0613, 1.0789, 1.0853):
        rng = np.random.default_rng(10)
        img1, img2, flow = _sample(rng, h, w)
        base = np.float32(1000 / sx)
        near = (base.view(np.int32) + np.arange(-40, 41)).astype(np.int32).view(np.float32)
        flow[:, :w // 2, 0] = near[rng.integers(0, len(near), (h, w // 2))]
        flow[:, :w // 2, 1] = -near[rng.integers(0, len(near), (h, w // 2))]
        flow[rng.uniform(size=(h, w)) < 0.01, 0] = np.nan
        flow[rng.uniform(size=(h, w)) < 0.01, 1] = np.inf
        flow[rng.uniform(size=(h, w)) < 0.01, 0] = -np.inf
        p0 = _P(M, crop, sx=sx, spatial=True, y0=3, x0=2)
        _, _, f, v = A.augment_dense(img1, img2, flow, p0)
        if planted(f, v).any():
            break
    else:
        raise AssertionError('no scale produced the planted threshold case')
    ps = [p0, _P(M, crop, sx=sx, spatial=True, hflip=True, vflip=True, y0=10, x0=30), _P(M, crop, hflip=True, y0=4, x0=8)]
    got = _check(M.FlowAugmentor(crop), [(img1, img2, flow)] * 3, ps, False)
    f, v = got[2][0], got[3][0]
    print(f'scale {sx}: {int(planted(f, v).sum())} pixels valid at |float32 flow| == 1000; '
          f'{int(np.isnan(f).sum())} NaN components')
    assert planted(f, v).any() and np.isnan(f).any() and (v == 0).any()


def test_kitti_dense_collisions(M):
    """A fully valid KITTI flow at downscales: many sources collide on each target and the last one wins; also a
    non-spatial sample (copy of flow and valid) and an h-flip."""
    rng = np.random.default_rng(11)
    aug = M.SparseFlowAugmentor(CROP_KITTI, do_flip=True)
    samples = [_sample(rng, *KITTI, sparse=True, density=1.01) for _ in range(3)]
    ps = [_P(M, CROP_KITTI, colour1=(BC, HSV), rects=[(1200, 300, 90, 99)], sx=0.78, spatial=True, y0=3, x0=1),
          _P(M, CROP_KITTI, sx=0.8317, spatial=True, hflip=True, y0=20, x0=40),
          _P(M, CROP_KITTI, hflip=True, y0=87, x0=282)]
    got = _check(aug, samples, ps, True)
    assert got[3][0].mean() > 0.9


def test_train_step_on_augmented_batch(M):
    import tf_raft_b200 as T
    from oracle import weights
    from tf_raft_b200.train import AdamW
    rng = np.random.default_rng(12)
    aug = M.FlowAugmentor((64, 96))
    np.random.seed(1)
    random.seed(2)
    batch = aug.batch([_sample(rng, 120, 160) for _ in range(2)])
    model = T.SmallRAFT(iters=2, iters_pred=2, precision='f16x2')
    model.load_params(weights.init_params('small', 3, bias_scale=0.05, norm_jitter=0.1))
    model.compile(optimizer=AdamW(weight_decay=1e-4, learning_rate=1e-4), clip_norm=1.0)
    out = model.train_step(batch)
    print(out)
    assert all(np.isfinite(float(v)) for v in out.values())
