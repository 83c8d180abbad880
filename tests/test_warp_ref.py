"""Flow warping and composition: the NumPy float32 restatement (oracle.warp_np) against float64 and torch's
grid_sample, composition identities, and the forward / backward chaining of RAFT.track_video on hand-made flows.
No GPU needed; tests/test_gpu_warp.py holds the kernels to this restatement bit for bit."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import warp_np

F32 = np.float32
EPS32 = float(np.finfo(F32).eps)


def landing_targets(n, size, rng):
    """n float32 landings on an axis of `size` texels: random, integer, half-integer, exactly size-1, one ulp past it,
    0, -0, just below 0, half a texel outside, +-inf and NaN."""
    last = F32(size - 1)
    special = np.array([0.0, -0.0, last, np.nextafter(last, F32(np.inf)), np.nextafter(last, F32(-np.inf)),
                        -2.0 ** -10, np.nextafter(F32(0), F32(-1)), -0.5, size - 0.5, np.inf, -np.inf, np.nan], F32)
    kind = rng.integers(0, 5, n)
    ints = rng.integers(0, size, n).astype(F32)
    p = rng.uniform(-0.1 * size - 1, 1.1 * size, n).astype(F32)
    p = np.where(kind == 1, ints, p)
    p = np.where(kind == 2, np.minimum(ints + F32(0.5), last), p)
    p = np.where(kind == 3, special[rng.integers(0, special.size, n)], p)
    return p


def flow_case(b, h, w, seed, hs=None, ws=None):
    """(B, H, W, 2) float32 flow whose landings on an (hs, ws) grid are `landing_targets`: f = p - x, exact for the
    small offsets, so x + f lands on the target where it matters (integers, the last texel and one ulp past it)."""
    hs, ws = hs or h, ws or w
    rng = np.random.default_rng(seed)
    gy, gx = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing='ij')
    px = landing_targets(b * h * w, ws, rng).reshape(b, h, w).astype(np.float64)
    py = landing_targets(b * h * w, hs, rng).reshape(b, h, w).astype(np.float64)
    with np.errstate(invalid='ignore'):
        return np.stack([px - gx, py - gy], -1).astype(F32)


def texels(b, h, w, c, seed, nonfinite=False):
    rng = np.random.default_rng(seed)
    t = rng.uniform(-4, 4, (b, h, w, c)).astype(F32)
    if nonfinite:
        flat = t.reshape(-1)
        idx = rng.choice(flat.size, max(1, flat.size // 50), replace=False)
        flat[idx] = rng.choice(np.array([np.nan, np.inf, -np.inf], F32), idx.size)
    return t


# --------------------------------------------------------------------------------------------- accuracy of the order
@pytest.mark.parametrize('shape', [(2, 9, 13, 3, 9, 13), (1, 1, 17, 2, 1, 17), (1, 11, 1, 1, 11, 1),
                                   (2, 7, 10, 4, 12, 5), (1, 40, 64, 8, 40, 64)])
@pytest.mark.parametrize('seed', [0, 1])
def test_float32_order_within_ulps_of_float64(shape, seed):
    """Bilinear warping in the header's float32 order stays within 4 ulps of float64 at the same (float32) landings,
    scaled by sum |weight * texel|; outside landings give the fill and occ in both."""
    b, h, w, c, hs, ws = shape
    flow = flow_case(b, h, w, seed, hs, ws)
    src = texels(b, hs, ws, c, seed + 10)
    got, occ = warp_np.warp(src, flow)
    want, occ64 = warp_np.warp(src, flow, dtype=np.float64)
    np.testing.assert_array_equal(occ, occ64)
    scale = warp_np.bilinear_weight_sum(src, flow)
    err = np.abs(got.astype(np.float64) - want)
    assert (err <= 4 * EPS32 * scale).all(), float((err / np.maximum(scale, 1e-300)).max() / EPS32)
    assert (got[occ] == 0).all() and occ.any() and (~occ).any()


def test_edge_landings_are_exact():
    """Integer landings, half-integers and the last texel take the texels the rule says, exactly."""
    src = texels(1, 6, 8, 2, 3)
    cases = {(0.0, 0.0): src[0, 0, 0], (7.0, 5.0): src[0, 5, 7], (3.0, 2.0): src[0, 2, 3],
             (2.5, 1.0): F32(0.5) * src[0, 1, 2] + F32(0.5) * src[0, 1, 3]}
    for (px, py), want in cases.items():
        flow = np.array([px, py], F32).reshape(1, 1, 1, 2)
        got, occ = warp_np.warp(src, flow)
        assert not occ.any()
        np.testing.assert_array_equal(got[0, 0, 0], np.asarray(want, F32))
    for px, py in ((np.nextafter(F32(7), F32(8)), 0), (0, np.nextafter(F32(5), F32(6))), (-1e-30, 0), (np.nan, 0),
                   (np.inf, 0), (0, -np.inf)):
        got, occ = warp_np.warp(src, np.array([px, py], F32).reshape(1, 1, 1, 2), fill=-7)
        assert occ.all() and (got == -7).all()
    # nearest: floor(p + 0.5), the half rounds up, clamped to the last texel
    for px, want_x in ((2.5, 3), (2.4999998, 2), (7.0, 7), (0.0, 0)):
        got, _ = warp_np.warp(src, np.array([px, 0], F32).reshape(1, 1, 1, 2), mode='nearest')
        np.testing.assert_array_equal(got[0, 0, 0], src[0, 0, want_x])


def test_nonfinite_texel_poisons_at_weight_zero():
    src = np.zeros((1, 2, 2, 1), F32)
    src[0, 0, 1, 0] = np.inf
    got, _ = warp_np.warp(src, np.zeros((1, 1, 1, 2), F32))          # landing (0, 0): weight of (0, 1) is 0
    assert np.isnan(got[0, 0, 0, 0])


@pytest.mark.parametrize('shape', [(2, 9, 13, 3, 9, 13), (1, 20, 31, 5, 14, 23)])
def test_bilinear_matches_grid_sample_strictly_inside(shape):
    """Where the landing is strictly inside, the kernel's rule is float64 F.grid_sample(align_corners=True) at the same
    positions, within the float32 bound."""
    b, h, w, c, hs, ws = shape
    rng = np.random.default_rng(5)
    gy, gx = np.meshgrid(np.arange(h), np.arange(w), indexing='ij')
    px = rng.uniform(0.01, ws - 1.01, (b, h, w)).astype(F32)
    py = rng.uniform(0.01, hs - 1.01, (b, h, w)).astype(F32)
    flow = np.stack([px - gx, py - gy], -1).astype(F32)
    src = texels(b, hs, ws, c, 6)
    got, occ = warp_np.warp(src, flow)
    assert not occ.any()
    qx, qy, _ = warp_np._landing(flow, hs, ws)                         # the float32 landings
    grid = torch.from_numpy(np.stack([2 * qx.astype(np.float64) / (ws - 1) - 1,
                                      2 * qy.astype(np.float64) / (hs - 1) - 1], -1))
    want = F.grid_sample(torch.from_numpy(src.astype(np.float64)).permute(0, 3, 1, 2), grid, mode='bilinear',
                         padding_mode='zeros', align_corners=True).permute(0, 2, 3, 1).numpy()
    scale = warp_np.bilinear_weight_sum(src, flow)
    assert (np.abs(got - want) <= 4 * EPS32 * scale + 1e-12).all()


# --------------------------------------------------------------------------------------------- composition
def test_compose_with_zero_second_flow_is_the_first():
    f1 = flow_case(2, 9, 13, 8)
    out, occ = warp_np.compose_flow(f1, np.zeros_like(f1))
    _, outside = warp_np.warp(np.zeros((2, 9, 13, 1), F32), f1)
    np.testing.assert_array_equal(occ, outside)
    np.testing.assert_array_equal(out.view(np.int32), f1.view(np.int32))       # bit for bit, NaN and -0 included


@pytest.mark.parametrize('t', [(3, -2), (0, 0), (-5, 4)])
def test_compose_integer_translation_is_the_sum_at_the_texel(t):
    b, h, w = 2, 10, 14
    f1 = np.broadcast_to(np.array(t, F32), (b, h, w, 2)).copy()
    f2 = texels(b, h, w, 2, 9)
    out, occ = warp_np.compose_flow(f1, f2)
    gy, gx = np.meshgrid(np.arange(h), np.arange(w), indexing='ij')
    inside = (gx + t[0] >= 0) & (gx + t[0] <= w - 1) & (gy + t[1] >= 0) & (gy + t[1] <= h - 1)
    np.testing.assert_array_equal(occ, np.broadcast_to(~inside, occ.shape))
    ys, xs = np.nonzero(inside)
    np.testing.assert_array_equal(out[:, ys, xs], f1[:, ys, xs] + f2[:, ys + t[1], xs + t[0]])
    np.testing.assert_array_equal(out[occ], f1[occ])


def test_compose_masks_and_nonfinite_results():
    b, h, w = 1, 6, 8
    f1 = np.full((b, h, w, 2), 1.0, F32)
    f2 = np.zeros((b, h, w, 2), F32)
    f2[0, 3, 3] = np.nan              # a corner of the landings of (1..2, 1..2), at weight 0 for three of them: lost
    occ1 = np.zeros((b, h, w), bool)
    occ1[0, 0, 0] = True
    occ2 = np.zeros((b, h, w), bool)
    occ2[0, 4, 5] = True                                    # reached from (4, 3)
    out, occ = warp_np.compose_flow(f1, f2, occ1, occ2)
    want = np.zeros((b, h, w), bool)
    want[0, :, w - 1] = want[0, h - 1, :] = True           # landing outside
    want[0, 0, 0] = want[0, 3, 4] = True
    want[0, 1:3, 1:3] = True
    np.testing.assert_array_equal(occ, want)
    np.testing.assert_array_equal(out[occ], f1[occ])
    assert np.isfinite(out).all()


# --------------------------------------------------------------------------------------------- chaining
def _band(h, w, band):
    return np.broadcast_to((np.arange(w) >= band[0]) & (np.arange(w) < band[1]), (h, w))


def _square_clip(n, h, w, size, v, band):
    """A size x size square at rows 3.. moving right by v px per frame over a static background, with the flows and
    masks a perfect estimator gives for each pair (t-1, t): F_{t-1->t} is v on the square, 0 elsewhere; occ_fw marks the
    background of frame t-1 that the square covers in frame t; B_{t->t-1} is -v on the square; occ_bw marks the
    background of frame t that the square uncovers.  Both masks also hold a static occluder band of columns."""
    fw, ofw, bw, obw = [], [], [], []
    rows = slice(3, 3 + size)
    for t in range(1, n):
        x0p, x0 = 2 + v * (t - 1), 2 + v * t
        f = np.zeros((1, h, w, 2), F32)
        f[0, rows, x0p:x0p + size, 0] = v
        o = _band(h, w, band)[None].copy()
        o[0, rows, x0p + size:x0 + size] = True
        g = np.zeros((1, h, w, 2), F32)
        g[0, rows, x0:x0 + size, 0] = -v
        ob = _band(h, w, band)[None].copy()
        ob[0, rows, x0p:x0] = True
        fw.append(f), ofw.append(o), bw.append(g), obw.append(ob)
    return fw, ofw, bw, obw


def test_forward_chaining_follows_the_square_and_keeps_lost_pixels_lost():
    """Frame 0's square moves v*t and stays tracked; the background it runs over is lost from the step it is covered
    on, for good, as is the band."""
    n, h, w, size, v = 6, 12, 30, 4, 2
    band = (24, 26)
    fw, ofw, _, _ = _square_clip(n, h, w, size, v, band)
    tracks = warp_np.track_forward(fw, ofw)
    assert len(tracks) == n - 1
    prev = np.zeros((1, h, w), bool)
    for t, (acc, lost) in enumerate(tracks, start=1):
        np.testing.assert_array_equal(acc[0, 3:3 + size, 2:2 + size, 0], np.full((size, size), v * t, F32))
        want = _band(h, w, band).copy()
        want[3:3 + size, 2 + size:2 + size + v * t] = True
        np.testing.assert_array_equal(lost[0], want)
        np.testing.assert_array_equal(acc[lost], fw[0][lost])            # lost background never moved: flow 0
        assert (lost >= prev).all()
        prev = lost


def test_pan_pushes_pixels_out_and_they_stay_lost():
    """A camera pan of +s px per frame: pixel x of frame 0 is at x + s*t; from the first t with x + s*t > W-1 it is
    lost for good, and its flow keeps its last in-frame value (the pair's own flow when lost at t = 1)."""
    n, h, w, s = 6, 4, 16, 3
    fw = [np.broadcast_to(np.array([s, 0], F32), (1, h, w, 2)).copy() for _ in range(n - 1)]
    ofw = [np.broadcast_to(np.arange(w) + s > w - 1, (1, h, w)).copy() for _ in range(n - 1)]
    tracks = warp_np.track_forward(fw, ofw)
    x = np.arange(w)
    kept = s * np.maximum((w - 1 - x) // s, 1)
    for t, (acc, lost) in enumerate(tracks, start=1):
        want_lost = x + s * t > w - 1
        np.testing.assert_array_equal(lost[0], np.broadcast_to(want_lost, (h, w)))
        np.testing.assert_array_equal(acc[0, 0, :, 0], np.where(want_lost, kept, s * t).astype(F32))


def test_backward_chaining_carries_labels_from_frame_zero():
    """Backward chaining of the same clip: frame t's square points back to frame 0's square, so nearest warping of
    frame 0's labels paints the square where it is in frame t; the background it uncovered and the band are lost."""
    n, h, w, size, v = 6, 12, 30, 4, 2
    band = (26, 28)
    _, _, bw, obw = _square_clip(n, h, w, size, v, band)
    labels = np.zeros((1, h, w, 1), np.uint8)
    labels[0, 3:3 + size, 2:2 + size] = 7
    for t, (acc, lost) in enumerate(warp_np.track_backward(bw, obw), start=1):
        moved, outside = warp_np.warp(labels, acc, mode='nearest')
        want = np.zeros((h, w), np.uint8)
        want[3:3 + size, 2 + v * t:2 + v * t + size] = 7
        want_lost = _band(h, w, band).copy()
        want_lost[3:3 + size, 2:2 + v * t] = True
        np.testing.assert_array_equal(lost[0], want_lost)
        np.testing.assert_array_equal(np.where(lost[0], 0, moved[0, ..., 0]), want)
        assert not outside.any()
