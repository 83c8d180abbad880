"""NumPy restatement of tf_raft/datasets/augmentor.py given its random parameters (test infrastructure, free of cv2).

What the CUDA kernels (tf_raft_b200/csrc/augment.cuh) must match bit for bit:
  * `resize_u8` / `resize_f32`: cv2.resize(..., fx, fy, INTER_LINEAR) on 3-channel uint8 and 2-channel float32.
    Output size rint(W*fx).  Source coordinate f = float32((d + 0.5) * (1/fx) - 0.5), s = floor(f), f -= s.  x clamps
    to the edge pixel with weight 0 outside the image; y does not clamp its weights (the border rows blend the clamped
    row with itself).  uint8: weights rint(w*2048), exact integer horizontal pass, then cv2's vectorised vertical
    rounding ((S0>>4)*b0 >> 16) + ((S1>>4)*b1 >> 16) + 2) >> 2.  cv2 keeps its scalar rounding for a row tail too
    short for a vector, so below ~24 output columns a few bytes differ; the augmentor never resizes that narrow.
    float32: one rounding per operation, no FMA; a column whose left tap is the last source column is S*1.
  * `rgb2hsv` / `hsv2rgb`: cv2.cvtColor(RGB2HSV / HSV2RGB) on uint8.  cv2 converts each image row in blocks of
    HSV_BLOCK = 32 pixels (4 float32 vectors of its x86 AVX2 dispatch, also taken on AVX-512 CPUs) and the last
    W mod 32 pixels of every row with a scalar loop: HSV->RGB truncates in the blocks and rounds to nearest even in
    that row tail, from the same float32 table.
  * the albumentations 0.4.6 LUTs, the eraser, the flips, the crops and `resize_sparse_flow_map`.  `bc_lut` and
    `hsv_luts` are transcriptions of albumentations 0.4.6 (which is not installed where this runs), as are the package's
    own copies in tf_raft_b200/datasets/augmentor.py; the GPU tests hold the kernels to these LUTs, and
    tests/test_augment_ref.py checks their NumPy casting against explicit float32 / float64 arithmetic.
`reference_draws` is a literal transcription of the reference's random draw calls, for the sampler test.
"""
import random

import numpy as np

F32, F64 = np.float32, np.float64


# ------------------------------------------------------------------------------------------------ resize
def resize_size(n, scale):
    """cv2's output size: saturate_cast<int>(n * scale), round half to even."""
    return int(np.rint(F64(n) * F64(scale)))


def _taps(n_src, n_dst, scale):
    """Per output index: (s0, s1, w0, w1, two_term) in float32 weights, before the caller's clamping rule."""
    inv = F64(1.0) / F64(scale)
    d = np.arange(n_dst, dtype=F64)
    f = ((d + 0.5) * inv - 0.5).astype(F32)
    s = np.floor(f)
    f = (f - s).astype(F32)
    return s.astype(np.int64), f


def _x_taps(n_src, n_dst, scale):
    s, f = _taps(n_src, n_dst, scale)
    two = s < n_src - 1                                    # cv2's xmax: from here on D = S[sx] * ONE
    f = np.where((s < 0) | (s >= n_src - 1), F32(0), f).astype(F32)
    s = np.clip(s, 0, n_src - 1)
    return s, np.minimum(s + 1, n_src - 1), (F32(1) - f).astype(F32), f, two


def _y_taps(n_src, n_dst, scale):
    s, f = _taps(n_src, n_dst, scale)
    return np.clip(s, 0, n_src - 1), np.clip(s + 1, 0, n_src - 1), (F32(1) - f).astype(F32), f


def _fix(w):
    return np.rint(w.astype(F32) * F32(2048)).astype(np.int64)


def resize_u8(img, fx, fy):
    """cv2.resize(img, None, fx=fx, fy=fy, interpolation=cv2.INTER_LINEAR) for (H, W, C) uint8."""
    h, w = img.shape[:2]
    oh, ow = resize_size(h, fy), resize_size(w, fx)
    x0, x1, a0, a1, _ = _x_taps(w, ow, fx)
    y0, y1, b0, b1 = _y_taps(h, oh, fy)
    src = img.astype(np.int64)
    hor = src[:, x0] * _fix(a0)[None, :, None] + src[:, x1] * _fix(a1)[None, :, None]      # exact integers
    ib0, ib1 = _fix(b0)[:, None, None], _fix(b1)[:, None, None]
    out = (((hor[y0] >> 4) * ib0) >> 16) + (((hor[y1] >> 4) * ib1) >> 16)
    return np.clip((out + 2) >> 2, 0, 255).astype(np.uint8)


def resize_f32(img, fx, fy):
    """cv2.resize(img, None, fx=fx, fy=fy, interpolation=cv2.INTER_LINEAR) for (H, W, C) float32."""
    img = np.asarray(img, dtype=F32)
    h, w = img.shape[:2]
    oh, ow = resize_size(h, fy), resize_size(w, fx)
    x0, x1, a0, a1, two = _x_taps(w, ow, fx)
    y0, y1, b0, b1 = _y_taps(h, oh, fy)
    with np.errstate(invalid='ignore', over='ignore'):
        hor = np.where(two[None, :, None], img[:, x0] * a0[None, :, None] + img[:, x1] * a1[None, :, None],
                       img[:, x0] * F32(1)).astype(F32)
        out = hor[y0] * b0[:, None, None] + hor[y1] * b1[:, None, None]
    assert out.dtype == F32
    return out


# ------------------------------------------------------------------------------------------------ colour
_HSV_SHIFT = 12
_SDIV = np.array([0] + [int(np.rint((255 << _HSV_SHIFT) / (1.0 * i))) for i in range(1, 256)], dtype=np.int64)
_HDIV = np.array([0] + [int(np.rint((180 << _HSV_SHIFT) / (6.0 * i))) for i in range(1, 256)], dtype=np.int64)
_SECTOR = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])   # (b, g, r) table entries


def rgb2hsv(img):
    """cv2.cvtColor(img, cv2.COLOR_RGB2HSV) for uint8 (hsv_shift = 12 fixed point, H in [0, 180])."""
    img = img.astype(np.int64)
    r, g, b = img[..., 0], img[..., 1], img[..., 2]
    v = np.maximum(np.maximum(r, g), b)
    diff = v - np.minimum(np.minimum(r, g), b)
    s = (diff * _SDIV[v] + (1 << (_HSV_SHIFT - 1))) >> _HSV_SHIFT
    h = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = (h * _HDIV[diff] + (1 << (_HSV_SHIFT - 1))) >> _HSV_SHIFT
    h = np.where(h < 0, h + 180, h)
    return np.stack([h, s, v], -1).astype(np.uint8)


def _fma1(a, b):
    """float32 fma(a, b, 1) rounded once: a*b is exact in float64; a float64 sum that lands on a float32 midpoint is
    moved by the sum's rounding error before the final rounding."""
    p = a.astype(F64) * b.astype(F64)
    s = p + 1.0
    err = (1.0 - (s - p)) + (p - (s - (s - p)))           # TwoSum error of p + 1
    r = s.astype(F32)
    mid = (s - r.astype(F64)) * 2.0
    ulp = np.spacing(np.abs(r)).astype(F64)
    tie = (np.abs(mid) == ulp) & (err != 0)
    adj = np.nextafter(s, np.where(err > 0, np.inf, -np.inf)).astype(F32)
    return np.where(tie, adj, r).astype(F32)


HSV_BLOCK = 32


def hsv2rgb(img):
    """cv2.cvtColor(img, cv2.COLOR_HSV2RGB) for (..., W, 3) uint8 with H < 180: float32 in [0, 1], times 255, truncated
    back to uint8, except in the last W mod HSV_BLOCK columns, where cv2's scalar row tail rounds half to even."""
    h, s, v = (img[..., k].astype(F32) for k in range(3))
    s, v = s * F32(1 / 255), v * F32(1 / 255)
    hs = h * F32(6 / 180)
    sec = np.floor(hs)
    f = hs - sec
    one = F32(1)
    tab = np.stack([v, v * (one - s), v * _fma1(-s, f), v * _fma1(-s, one - f)], -1)
    idx = _SECTOR[sec.astype(np.int64) % 6]
    rgb = np.stack([np.take_along_axis(tab, idx[..., k:k + 1], -1)[..., 0] for k in (2, 1, 0)], -1)
    rgb = rgb * F32(255)
    w = img.shape[-2]
    tail = (np.arange(w) >= w - w % HSV_BLOCK)[:, None]
    return np.clip(np.where(tail, np.rint(rgb), np.trunc(rgb)), 0, 255).astype(np.uint8)


def bc_lut(alpha, beta):
    """albumentations 0.4.6 _brightness_contrast_adjust_uint (brightness_by_max=True) as a 256-entry uint8 LUT."""
    lut = np.arange(0, 256).astype('float32')
    if alpha != 1:
        lut *= alpha
    if beta != 0:
        lut += beta * 255
    return np.clip(lut, 0, 255).astype(np.uint8)


def hsv_luts(hue_shift, sat_shift, val_shift):
    """albumentations 0.4.6 _shift_hsv_uint8's three LUTs (hue, sat, val)."""
    lut = np.arange(0, 256, dtype=np.int16)
    return (np.mod(lut + hue_shift, 180).astype(np.uint8), np.clip(lut + sat_shift, 0, 255).astype(np.uint8),
            np.clip(lut + val_shift, 0, 255).astype(np.uint8))


def colour(img, bc, hsv):
    """RandomBrightnessContrast (bc = (alpha, beta) or None) then HueSaturationValue (hsv = shifts or None)."""
    if bc is not None:
        img = bc_lut(*bc)[img]
    if hsv is not None:
        hl, sl, vl = hsv_luts(*hsv)
        x = rgb2hsv(img)
        img = hsv2rgb(np.stack([hl[x[..., 0]], sl[x[..., 1]], vl[x[..., 2]]], -1))
    return img


def eraser(img2, rects):
    """augmentor.py:61-74: each (x0, y0, dx, dy) rectangle, clipped by slicing, set to the truncated channel mean."""
    img2 = img2.copy()
    if rects:
        mean = np.mean(img2.reshape(-1, 3), axis=0)
        for x0, y0, dx, dy in rects:
            img2[y0:y0 + dy, x0:x0 + dx, :] = mean
    return img2


# ------------------------------------------------------------------------------------------------ whole samples
def augment_dense(img1, img2, flow, p):
    """FlowAugmentor.__call__ given its parameters `p` (see tf_raft_b200.datasets.augmentor.DenseParams), then
    dataset.py:102's valid on the float64 flow and the final float32 cast.  -> (img1, img2, flow f32, valid f32)."""
    img1 = colour(img1, *p.colour1)
    img2 = colour(img2, *p.colour2)
    img2 = eraser(img2, p.rects)
    if p.spatial:
        img1 = resize_u8(img1, p.scale_x, p.scale_y)
        img2 = resize_u8(img2, p.scale_x, p.scale_y)
        flow = resize_f32(flow, p.scale_x, p.scale_y)
        flow = flow * [p.scale_x, p.scale_y]
    if p.hflip:
        img1, img2 = img1[:, ::-1], img2[:, ::-1]
        flow = flow[:, ::-1] * [-1.0, 1.0]
    if p.vflip:
        img1, img2 = img1[::-1, :], img2[::-1, :]
        flow = flow[::-1, :] * [1.0, -1.0]
    ch, cw = p.crop
    sl = np.s_[p.y0:p.y0 + ch, p.x0:p.x0 + cw]
    img1, img2, flow = img1[sl], img2[sl], flow[sl]
    with np.errstate(invalid='ignore'):
        valid = (np.abs(flow[:, :, 0]) < 1000) * (np.abs(flow[:, :, 1]) < 1000)
    return (np.ascontiguousarray(img1), np.ascontiguousarray(img2), np.ascontiguousarray(flow, dtype=F32),
            valid.astype(F32))


def resize_sparse_flow_map(flow, valid, fx=1.0, fy=1.0):
    """augmentor.py:183-215, verbatim."""
    ht, wd = flow.shape[:2]
    coords = np.meshgrid(np.arange(wd), np.arange(ht))
    coords = np.stack(coords, axis=-1)
    coords = coords.reshape(-1, 2).astype(np.float32)
    flow = flow.reshape(-1, 2).astype(np.float32)
    valid = valid.reshape(-1).astype(np.float32)
    coords0 = coords[valid >= 1]
    flow0 = flow[valid >= 1]
    ht1 = int(round(ht * fy))
    wd1 = int(round(wd * fx))
    coords1 = coords0 * [fx, fy]
    flow1 = flow0 * [fx, fy]
    xx = np.round(coords1[:, 0]).astype(np.int32)
    yy = np.round(coords1[:, 1]).astype(np.int32)
    v = (xx > 0) & (xx < wd1) & (yy > 0) & (yy < ht1)
    xx = xx[v]
    yy = yy[v]
    flow1 = flow1[v]
    flow_img = np.zeros([ht1, wd1, 2], dtype=np.float32)
    valid_img = np.zeros([ht1, wd1], dtype=np.int32)
    flow_img[yy, xx] = flow1
    valid_img[yy, xx] = 1
    return flow_img, valid_img


def augment_sparse(img1, img2, flow, valid, p):
    """SparseFlowAugmentor.__call__ given its parameters `p` -> (img1, img2, flow f32, valid f32)."""
    img1 = colour(img1, *p.colour1)
    img2 = colour(img2, *p.colour2)
    img2 = eraser(img2, p.rects)
    if p.spatial:
        img1 = resize_u8(img1, p.scale_x, p.scale_y)
        img2 = resize_u8(img2, p.scale_x, p.scale_y)
        flow, valid = resize_sparse_flow_map(flow, valid, fx=p.scale_x, fy=p.scale_y)
    if p.hflip:
        img1, img2 = img1[:, ::-1], img2[:, ::-1]
        flow = flow[:, ::-1] * [-1.0, 1.0]
        valid = valid[:, ::-1]
    ch, cw = p.crop
    sl = np.s_[p.y0:p.y0 + ch, p.x0:p.x0 + cw]
    return (np.ascontiguousarray(img1[sl]), np.ascontiguousarray(img2[sl]),
            np.ascontiguousarray(flow[sl], dtype=F32), np.ascontiguousarray(valid[sl], dtype=F32))


# ------------------------------------------------------------------------------------------------ the draws
def _photo_aug_draws(bc_limit, hsv_limits):
    """albumentations 0.4.6 Compose([RandomBrightnessContrast, HueSaturationValue]) (p = 1, each p = 0.5): the calls of
    core/composition.py Compose.__call__, core/transforms_interface.py BasicTransform.__call__ and the two get_params."""
    out = []
    random.random()                                            # Compose: random.random() < self.p
    if random.random() < 0.5:                                  # RandomBrightnessContrast
        alpha = 1.0 + random.uniform(-bc_limit, bc_limit)
        beta = 0.0 + random.uniform(-bc_limit, bc_limit)
        out.append(('bc', alpha, beta))
    if random.random() < 0.5:                                  # HueSaturationValue
        out.append(('hsv', random.uniform(-hsv_limits[0], hsv_limits[0]),
                    random.uniform(-hsv_limits[1], hsv_limits[1]), random.uniform(-hsv_limits[2], hsv_limits[2])))
    return out


def reference_draws(kind, ht, wd, crop_size, min_scale=-0.2, max_scale=0.5, do_flip=None):
    """Every random value augmentor.py draws for one (ht, wd) sample, in its call order, as a flat list of tuples."""
    out = []
    if kind == 'dense':
        do_flip = True if do_flip is None else do_flip
        limits = (0.4, (int(0.5 / 3.14 * 180), int(0.4 * 255), int(0.)))
        if np.random.rand() < 0.2:
            out.append(('asym', True))
            out += _photo_aug_draws(*limits)
            out.append(('img2',))
            out += _photo_aug_draws(*limits)
        else:
            out.append(('asym', False))
            out += _photo_aug_draws(*limits)
    else:
        do_flip = False if do_flip is None else do_flip
        out += _photo_aug_draws(0.3, (int(0.3 / 3.14 * 180), int(0.3 * 255), int(0.)))
    if np.random.rand() < 0.5:
        for _ in range(np.random.randint(1, 3)):
            x0 = np.random.randint(0, wd)
            y0 = np.random.randint(0, ht)
            dx = np.random.randint(50, 100)
            dy = np.random.randint(50, 100)
            out.append(('rect', x0, y0, dx, dy))
    pad = 8 if kind == 'dense' else 1
    min_s = np.maximum((crop_size[0] + pad) / float(ht), (crop_size[1] + pad) / float(wd))
    scale = 2 ** np.random.uniform(min_scale, max_scale)
    scale_x = scale
    scale_y = scale
    if kind == 'dense' and np.random.rand() < 0.8:
        scale_x *= 2 ** np.random.uniform(-0.2, 0.2)
        scale_y *= 2 ** np.random.uniform(-0.2, 0.2)
    scale_x = np.clip(scale_x, min_s, None)
    scale_y = np.clip(scale_y, min_s, None)
    spatial = np.random.rand() < 0.8
    out.append(('scale', float(scale_x), float(scale_y), bool(spatial)))
    h1, w1 = (int(np.rint(ht * scale_y)), int(np.rint(wd * scale_x))) if spatial else (ht, wd)
    if kind == 'dense':
        if do_flip:
            out.append(('flip', bool(np.random.rand() < 0.5), bool(np.random.rand() < 0.1)))
        y0 = np.random.randint(0, h1 - crop_size[0])
        x0 = np.random.randint(0, w1 - crop_size[1])
    else:
        if do_flip:
            out.append(('flip', bool(np.random.rand() < 0.5), False))
        y0 = np.random.randint(0, h1 - crop_size[0] + 20)
        x0 = np.random.randint(-50, w1 - crop_size[1] + 50)
        y0 = np.clip(y0, 0, h1 - crop_size[0])
        x0 = np.clip(x0, 0, w1 - crop_size[1])
    out.append(('crop', int(y0), int(x0)))
    return out
