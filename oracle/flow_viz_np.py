"""NumPy restatement of tf_raft/datasets/flow_viz.py (the Middlebury colour wheel) as the GPU computes it.

Every step is written with the dtype NumPy 2 gives the reference's expression (NEP 50: a Python scalar takes the array's
dtype; a float32 array minus an int32 array is float64), one ufunc per operation, so no step is fused.  The one
deliberate difference from the reference as run: atan2 is `float32(np.arctan2(float64, float64))`, the correctly rounded
float32 value, where NumPy's own float32 arctan2 depends on the build (its AVX-512 loop is off by one ulp on about a
third of inputs).  `near` marks the pixels whose float64 atan2 lies within 2^-44 relative of a float32 rounding
midpoint: only there may two correct float64 atan2 implementations round to different float32 values.

`golden_cases()` regenerates the inputs of tests/golden/flow_viz.npz from seeds.
"""
import numpy as np

WHEEL_SEGMENTS = (('RY', 15), ('YG', 6), ('GC', 4), ('CB', 11), ('BM', 13), ('MR', 6))
NEAR_REL = 2.0 ** -44


def make_colorwheel():
    """(55, 3) float64 table: six ramps between red, yellow, green, cyan, blue and magenta, each ramp step
    floor(255 * j / n) (Baker et al., ICCV 2007)."""
    rows = []
    for name, n in WHEEL_SEGMENTS:
        for j in range(n):
            up, down = (255 * j) // n, 255 - (255 * j) // n
            rows.append({'RY': (255, up, 0), 'YG': (down, 255, 0), 'GC': (0, 255, up),
                         'CB': (0, down, 255), 'BM': (up, 0, 255), 'MR': (255, 0, down)}[name])
    return np.array(rows, dtype=np.float64)


def near_midpoint(a64):
    """True where float64 `a64` lies within NEAR_REL relative of a float32 rounding midpoint."""
    a32 = a64.astype(np.float32)
    with np.errstate(invalid='ignore'):
        other = np.where(a64 >= a32.astype(np.float64), np.nextafter(a32, np.float32(np.inf)),
                         np.nextafter(a32, np.float32(-np.inf)))
        mid = (a32.astype(np.float64) + other.astype(np.float64)) / 2
        return np.abs(a64 - mid) <= NEAR_REL * np.abs(a64)


def steps(u, v):
    """The intermediate arrays of flow_uv_to_colors for float32 u, v (names as in the reference)."""
    u = np.asarray(u, np.float32)
    v = np.asarray(v, np.float32)
    with np.errstate(invalid='ignore', over='ignore'):
        rad = np.sqrt(np.square(u) + np.square(v))                                   # float32
        a64 = np.arctan2((-v).astype(np.float64), (-u).astype(np.float64))
        a = a64.astype(np.float32) / np.float32(np.pi)                             # float32
        fk = (a + np.float32(1)) / np.float32(2) * np.float32(54)                    # float32
        bad = ~np.isfinite(fk)
        k0 = np.floor(np.where(bad, 0, fk)).astype(np.int32)
        k1 = k0 + 1
        k1[k1 == 55] = 0
        f = fk - k0                                                                  # float32 - int32: float64
    return dict(rad=rad, a64=a64, a=a, fk=fk, k0=k0, k1=k1, f=f, bad=bad)


def flow_uv_to_colors(u, v, convert_to_bgr=False):
    """(H, W) float32 u, v -> ((H, W, 3) uint8 image, (H, W) near-midpoint mask).  A pixel whose angle is NaN is
    (0, 0, 0), where the reference raises IndexError."""
    s = steps(u, v)
    wheel = make_colorwheel()
    img = np.zeros(s['rad'].shape + (3,), np.uint8)
    idx = s['rad'] <= 1
    for i in range(3):
        col0 = wheel[s['k0'], i] / 255.0
        col1 = wheel[s['k1'], i] / 255.0
        col = (1 - s['f']) * col0 + s['f'] * col1                                     # float64
        with np.errstate(invalid='ignore'):                                          # inf rad: both branches run
            col = np.where(idx, 1 - s['rad'] * (1 - col), col * 0.75)
            img[..., 2 - i if convert_to_bgr else i] = np.where(s['bad'], 0, np.floor(255 * col))
    return img, near_midpoint(s['a64'])


def flow_to_image(flow_uv, clip_flow=None, convert_to_bgr=False, rad_max=None):
    """(H, W, 2) float32 flow -> ((H, W, 3) uint8, near mask).  `rad_max` replaces the image's own maximum radius."""
    flow_uv = np.asarray(flow_uv, np.float32)
    if clip_flow is not None:
        flow_uv = np.clip(flow_uv, 0, np.float32(clip_flow))
    u, v = flow_uv[..., 0], flow_uv[..., 1]
    with np.errstate(over='ignore', invalid='ignore'):
        if rad_max is None:
            rad_max = np.max(np.sqrt(np.square(u) + np.square(v)))
        d = np.float32(rad_max) + np.float32(1e-5)                                   # float32 under NEP 50
        u, v = u / d, v / d
    return flow_uv_to_colors(u, v, convert_to_bgr)


def _smooth(rng, h, w, scale):
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    c = rng.uniform(-1, 1, 6)
    u = np.sin(x / w * 3 * c[0] + c[1]) + c[2] * (y / h - 0.5)
    v = np.cos(y / h * 3 * c[3] + c[4]) + c[5] * (x / w - 0.5)
    return (np.stack([u, v], -1) * scale + rng.standard_normal((h, w, 2)) * scale * 1e-3).astype(np.float32)


def golden_cases():
    """name -> (flow (H, W, 2) float32, kwargs of flow_to_image).  Seeded: the same arrays on every machine."""
    cases = {}
    for seed, (h, w) in enumerate([(1, 1), (1, 9), (7, 1), (3, 5), (17, 31), (40, 61)]):
        for scale in (1e-3, 1.0, 30.0, 1e4):
            rng = np.random.default_rng(1000 * seed + int(np.log10(scale) + 4))
            cases[f'rand_{h}x{w}_{scale:g}'] = ((rng.standard_normal((h, w, 2)) * scale).astype(np.float32), {})
    cases['sintel_436x1024'] = (_smooth(np.random.default_rng(7), 436, 1024, 20.0), {})
    rng = np.random.default_rng(8)
    cases['clip_24x40'] = ((rng.standard_normal((24, 40, 2)) * 10).astype(np.float32), dict(clip_flow=5.0))
    cases['bgr_24x40'] = ((rng.standard_normal((24, 40, 2)) * 10).astype(np.float32), dict(convert_to_bgr=True))
    cases['smooth_bgr_clip_96x128'] = (_smooth(rng, 96, 128, 8.0), dict(clip_flow=6.0, convert_to_bgr=True))
    cases['zero_4x6'] = (np.zeros((4, 6, 2), np.float32), {})
    cases['signed_zero_1x6'] = (np.array([[[5, 0], [5, -0.0], [-3, 0], [-3, -0.0], [0, 5], [-0.0, 5]]], np.float32), {})
    cases['overflow_1x4'] = (np.array([[[2e19, 1], [1, 1], [-3e19, 0], [0, -1]]], np.float32), {})
    axis = [[k, 0] for k in (1, 2, -4, 8)] + [[0, k] for k in (1, -2, 4, -8)]
    cases['axis_1x8'] = (np.array([axis], np.float32), {})
    return cases
