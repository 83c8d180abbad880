"""CPU checks of the training augmentation's restatement (oracle/augment_np.py) and of the host-side sampler.

Where OpenCV imports, the restatement's resize and RGB<->HSV equal cv2 bit for bit; the sampler, seeded, reproduces a
literal transcription of tf_raft/datasets/augmentor.py's draw calls; resize_sparse_flow_map's edge cases; a crop that
does not fit raises ValueError.
"""
import random

import numpy as np
import pytest

from oracle import augment_np as A

try:
    import cv2
except ImportError:          # the restatement is cv2-free; only the cross-checks need it
    cv2 = None

needs_cv2 = pytest.mark.skipif(cv2 is None, reason='OpenCV is not installed')


def _resize_cases():
    """>= 40 (h, w, fx, fy): random shapes and scales in 2^-0.3 .. 2^1, augmentor-like downscales at the min_scale clip
    ((crop + 8) / size of Chairs, Sintel and KITTI crops), stretched pairs; every output at least 32 columns wide."""
    rng = np.random.default_rng(2024)
    out = []
    while len(out) < 40:
        h, w = (int(v) for v in rng.integers(20, 401, 2))
        fx, fy = (float(v) for v in 2 ** rng.uniform(-0.3, 1.0, 2))
        if A.resize_size(w, fx) >= 32:
            out.append((h, w, fx, fy))
    for (h, w), (ch, cw) in (((384, 512), (368, 496)), ((436, 1024), (368, 768)), ((375, 1242), (288, 960))):
        s = max((ch + 8) / float(h), (cw + 8) / float(w))
        out += [(h, w, s, s), (h, w, s * 2 ** 0.13, s), (h, w, 2 ** -0.2, 2 ** 0.5)]
    return out


@needs_cv2
def test_resize_equals_cv2(record_property):
    """uint8 3-channel and float32 2-channel cv2.resize INTER_LINEAR, every byte and every float bit.  Outputs narrower
    than ~24 columns are a known difference (cv2's scalar row tail rounds differently) and are not asserted."""
    record_property('cv2_version', cv2.__version__)
    print(f'cv2 {cv2.__version__}')
    rng = np.random.default_rng(7)
    n = 0
    for h, w, fx, fy in _resize_cases():
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        flow = (rng.standard_normal((h, w, 2)) * 40).astype(np.float32)
        want = cv2.resize(img, None, fx=fx, fy=fy, interpolation=cv2.INTER_LINEAR)
        got = A.resize_u8(img, fx, fy)
        assert got.shape == want.shape and np.array_equal(got, want), (h, w, fx, fy)
        want = cv2.resize(flow, None, fx=fx, fy=fy, interpolation=cv2.INTER_LINEAR)
        got = A.resize_f32(flow, fx, fy)
        assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), (h, w, fx, fy)
        n += want.shape[0] * want.shape[1]
    print(f'{len(_resize_cases())} shapes, {n} output pixels bit-exact')


def _all_rgb():
    x = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([x >> 16, (x >> 8) & 255, x & 255], -1).astype(np.uint8).reshape(1 << 16, 256, 3)


@needs_cv2
def test_rgb2hsv_equals_cv2_all_colours(record_property):
    record_property('cv2_version', cv2.__version__)
    rgb = _all_rgb()
    assert np.array_equal(A.rgb2hsv(rgb), cv2.cvtColor(rgb, cv2.COLOR_RGB2HSV))


@needs_cv2
@pytest.mark.parametrize('width', [256, 1242, 1226, 611, 31])
def test_hsv2rgb_equals_cv2_all_valid_triples(width, record_property):
    """All 180 * 256 * 256 triples with H < 180 laid out in rows of `width` pixels (the remainder dropped): 256 has no
    row tail, 1242 and 1226 are KITTI widths whose last 26 / 10 columns are cv2's scalar tail, 611 an odd size, and in
    rows of 31 every pixel is in the tail."""
    record_property('cv2_version', cv2.__version__)
    hsv = _all_rgb().reshape(-1, 3)[:180 * 65536]
    hsv = hsv[:hsv.shape[0] // width * width].reshape(-1, width, 3)
    got, want = A.hsv2rgb(hsv), cv2.cvtColor(hsv, cv2.COLOR_HSV2RGB)
    bad = np.argwhere((got != want).any(-1))
    assert bad.size == 0, (len(bad), bad[:5].tolist())


@needs_cv2
def test_colour_equals_albumentations_path_at_kitti_width():
    """The symmetric colour path as albumentations 0.4.6 runs it with cv2 (LUT, cvtColor to HSV, three LUTs, cvtColor
    back) on a stacked (2H, 1242) image, against the restatement's `colour`."""
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (2 * 75, 1242, 3), dtype=np.uint8)
    for bc, hsv in (((1.23, -0.17), (-21.7, 88.4, 0.0)), (None, (27.9, -101.9, 0.0)), ((0.71, 0.3), (-3.2, 5.5, 0.0))):
        x = cv2.LUT(img, A.bc_lut(*bc)) if bc is not None else img
        h, s_, v = cv2.split(cv2.cvtColor(x, cv2.COLOR_RGB2HSV))
        hl, sl, vl = A.hsv_luts(*hsv)
        want = cv2.cvtColor(cv2.merge((cv2.LUT(h, hl), cv2.LUT(s_, sl), cv2.LUT(v, vl))), cv2.COLOR_HSV2RGB)
        assert np.array_equal(A.colour(img, bc, hsv), want)


def test_luts_follow_numpy_casting():
    """The LUT transcriptions against the arithmetic NumPy's casting implies: brightness/contrast in float32 (the Python
    float alpha cast to float32 before the multiply, beta * 255 formed in float64 then cast), hue / sat / val in
    float64, all truncated; and the package's copies equal the oracle's."""
    from tf_raft_b200.datasets import augmentor as G
    rng = np.random.default_rng(4)
    i32, i64 = np.arange(256, dtype=np.float32), np.arange(256, dtype=np.float64)
    for _ in range(500):
        alpha, beta = 1.0 + rng.uniform(-0.4, 0.4), rng.uniform(-0.4, 0.4)
        want = np.clip((i32 * np.float32(alpha)) + np.float32(beta * 255), 0, 255).astype(np.uint8)
        assert np.array_equal(A.bc_lut(alpha, beta), want) and np.array_equal(G.bc_lut(alpha, beta), want)
        hue, sat, val = rng.uniform(-28, 28), rng.uniform(-102, 102), rng.uniform(-5, 5)
        want = (np.fmod(np.fmod(i64 + hue, 180) + 180, 180).astype(np.uint8),
                np.clip(i64 + sat, 0, 255).astype(np.uint8), np.clip(i64 + val, 0, 255).astype(np.uint8))
        for got in (A.hsv_luts(hue, sat, val), G.hsv_luts(hue, sat, val)):
            assert all(np.array_equal(g, w) for g, w in zip(got, want))


def test_fma1_rounds_once():
    """The HSV->RGB fma emulation equals an exact rational fma on every (s, f) the conversion can meet."""
    from fractions import Fraction
    s = (np.arange(256, dtype=np.float32) * np.float32(1 / 255)).astype(np.float32)
    hs = (np.arange(180, dtype=np.float32) * np.float32(6 / 180)).astype(np.float32)
    f = (hs - np.floor(hs)).astype(np.float32)
    fs = np.unique(np.concatenate([f, (np.float32(1) - f).astype(np.float32)]))
    S, Fv = np.meshgrid(s, fs, indexing='ij')
    got = A._fma1(-S, Fv)
    grid = np.sort(np.unique(got))
    for a, b, g in zip(S.ravel()[::7], Fv.ravel()[::7], got.ravel()[::7]):
        exact = Fraction(1) - Fraction(float(a)) * Fraction(float(b))
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-1)), lo, np.nextafter(lo, np.float32(2))]
        best = min(cands, key=lambda c: (abs(Fraction(float(c)) - exact), int(np.float32(c).view(np.uint32)) & 1))
        assert g == best, (a, b, g, best)
    assert grid.size > 1


def _photo_draws(c):
    bc, hsv = c
    out = []
    if bc is not None:
        out.append(('bc',) + tuple(bc))
    if hsv is not None:
        out.append(('hsv',) + tuple(hsv))
    return out


def _as_draws(p, kind, asym, do_flip):
    out = [('asym', asym)] if kind == 'dense' else []
    out += _photo_draws(p.colour1)
    if asym:
        out += [('img2',)] + _photo_draws(p.colour2)
    out += [('rect',) + tuple(r) for r in p.rects]
    out.append(('scale', p.scale_x, p.scale_y, p.spatial))
    if do_flip:
        out.append(('flip', p.hflip, p.vflip))
    out.append(('crop', p.y0, p.x0))
    return out


@pytest.mark.parametrize('kind,crop,shapes,do_flip', [
    ('dense', (368, 496), [(384, 512), (436, 1024)], True),
    ('dense', (256, 320), [(300, 400)], False),
    ('sparse', (288, 960), [(375, 1242), (370, 1226)], False),
    ('sparse', (288, 960), [(375, 1242)], True),
])
def test_sampler_reproduces_reference_draws(kind, crop, shapes, do_flip):
    """1000 samples each: the sampler and the transcription, started from the same seeds of np.random and random, give
    the same values and leave both generators in the same state after every sample."""
    from tf_raft_b200.datasets import FlowAugmentor, SparseFlowAugmentor
    aug = (FlowAugmentor if kind == 'dense' else SparseFlowAugmentor)(crop, do_flip=do_flip, device='cpu')
    np.random.seed(11)
    random.seed(12)
    for i in range(1000):
        ht, wd = shapes[i % len(shapes)]
        st_np, st_py = np.random.get_state(), random.getstate()
        want = A.reference_draws(kind, ht, wd, crop, do_flip=do_flip)
        end_np, end_py = np.random.get_state(), random.getstate()
        np.random.set_state(st_np)
        random.setstate(st_py)
        p = aug.sample_params(ht, wd)
        asym = kind == 'dense' and want[0][1]
        assert _as_draws(p, kind, asym, do_flip) == want, i
        assert random.getstate() == end_py
        s1, s2 = np.random.get_state(), end_np
        assert s1[0] == s2[0] and np.array_equal(s1[1], s2[1]) and s1[2:] == s2[2:]


def test_too_small_source_raises():
    """A source the crop does not fit: the reference's np.random.randint(0, <= 0) raises ValueError, and so does the
    sampler whenever the spatial branch is not taken (a resize always leaves crop + 8 / + 1)."""
    from tf_raft_b200.datasets import FlowAugmentor, SparseFlowAugmentor
    np.random.seed(0)
    random.seed(0)
    for aug, (h, w) in ((FlowAugmentor((368, 496), device='cpu'), (368, 600)),
                        (SparseFlowAugmentor((288, 960), device='cpu'), (200, 1000))):
        with pytest.raises(ValueError):
            for _ in range(100):
                aug.sample_params(h, w)


def test_sparse_map_edge_cases():
    """resize_sparse_flow_map: colliding targets go to the last source in index order; column and row 0 are dropped by
    the strict > 0 bound; .5 coordinates round half to even."""
    h, w = 4, 6
    flow = np.arange(h * w * 2, dtype=np.float32).reshape(h, w, 2)
    valid = np.ones((h, w), np.float32)
    # fx = fy = 0.5: x in {0..5} -> 0, 0.5 -> 0, 1, 1.5 -> 2, 2, 2.5 -> 2: targets 0 (x 0, 1), 1 (x 2), 2 (x 3, 4, 5)
    f, v = A.resize_sparse_flow_map(flow, valid, 0.5, 0.5)
    assert f.shape == (2, 3, 2) and v.shape == (2, 3)
    # row yy = 1 gets y in {2, 3} (y = 1 -> 0.5 -> 0 is dropped, y = 3 -> 1.5 -> 2 is out of range): only y = 2
    assert v.tolist() == [[0, 0, 0], [0, 1, 1]]
    assert f[1, 1].tolist() == list(flow[2, 2] * 0.5)                 # x = 2 -> 1.0 (x = 1 -> 0.5 -> 0 dropped)
    assert f[1, 2].tolist() == list(flow[2, 5] * 0.5)                 # x = 3, 4, 5 -> 2: the last (x = 5) wins
    # an invalid source never lands
    valid[2, 5] = 0
    f, v = A.resize_sparse_flow_map(flow, valid, 0.5, 0.5)
    assert f[1, 2].tolist() == list(flow[2, 4] * 0.5)
    # fx = 1.5: x = 1 -> 1.5 -> 2, x = 3 -> 4.5 -> 4, x = 5 -> 7.5 -> 8 (half to even); x = 0 -> 0 dropped
    f, v = A.resize_sparse_flow_map(flow, np.ones((h, w), np.float32), 1.5, 1.0)
    assert v[1].tolist() == [0, 0, 1, 1, 1, 0, 1, 0, 1]
    assert f[1, 2].tolist() == list((flow[1, 1].astype(np.float64) * [1.5, 1.0]).astype(np.float32))
    assert f[1, 4].tolist() == list((flow[1, 3].astype(np.float64) * [1.5, 1.0]).astype(np.float32))
    assert v[0].sum() == 0 and v[:, 0].sum() == 0
