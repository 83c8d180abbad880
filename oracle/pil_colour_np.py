"""NumPy restatement of torchvision's ColorJitter on an RGB PIL image (test infrastructure, free of PIL).

RAFT's augmentor (core/utils/augmentor.py) jitters with torchvision's ColorJitter on PIL images: the four ops run in
the order `fn_idx = torch.randperm(4)` draws, each through Pillow's C code.  This module states that arithmetic one
rounded operation at a time, in the order the CUDA kernels (tf_raft_b200/csrc/colour.cuh) evaluate it;
tests/test_colour_jitter_ref.py holds it to Pillow over every input of each conversion.

  * blend (ImageEnhance's Image.blend(degenerate, img, f)): the float32 `a + f*(b - a)` with f = float32(factor), one
    multiply and one add (no FMA), clipped to [0, 255] and truncated.
  * RGB->L: (19595 R + 38470 G + 7471 B + 0x8000) >> 16.
  * brightness: blend towards 0.  contrast: blend towards m = int(sum(L) / n + 0.5), the double-precision mean of the
    image's L at that point of the sequence.  saturation: blend towards the pixel's own L.
  * hue: Pillow's RGB->HSV, H += uint8(int32(hue * 255)) with wraparound, Pillow's HSV->RGB.  The round trip runs even
    when the byte is 0.  Pillow's conversions mix float32 and float64 the way C promotes them: see `rgb_to_hsv` and
    `hsv_to_rgb`.
"""
import numpy as np

F32, F64 = np.float32, np.float64
BRIGHTNESS, CONTRAST, SATURATION, HUE = 0, 1, 2, 3


def blend(a, b, factor):
    """Image.blend(a, b, factor) on uint8: fl32(a + fl32(f * (b - a))), f = float32(factor), clipped and truncated."""
    f = F32(factor)
    d = (np.asarray(b, np.int32) - np.asarray(a, np.int32)).astype(F32)
    t = (np.asarray(a, np.int32).astype(F32) + (f * d).astype(F32)).astype(F32)
    return np.clip(np.trunc(t), 0, 255).astype(np.uint8)


def rgb_to_l(rgb):
    """Image.convert('L') of (..., 3) uint8."""
    x = np.asarray(rgb, np.int64)
    return ((19595 * x[..., 0] + 38470 * x[..., 1] + 7471 * x[..., 2] + 0x8000) >> 16).astype(np.uint8)


def contrast_mean(l_sum, n):
    """ImageEnhance.Contrast's grey level: int(sum / n + 0.5) in float64 (ImageStat's mean)."""
    return int(F64(l_sum) / F64(n) + F64(0.5))


def hue_byte(hue_factor):
    """torchvision adjust_hue's shift: np.int32(hue_factor * 255).astype(np.uint8), a truncation then a wrap."""
    return int(np.int32(hue_factor * 255).astype(np.uint8))


def rgb_to_hsv(rgb):
    """Pillow's RGB->HSV on (..., 3) uint8.  float32: cr = max - min, s = cr / max, rc, gc, bc = (max - c) / cr.
    float64: the hue sum (2.0 and 4.0 are doubles), rounded to float32, then h = fl32(fmod(h / 6.0 + 1.0, 1.0));
    H = int(h * 255.0), S = int(s * 255.0) in float64, truncated.  A grey pixel is (0, 0, v)."""
    x = np.asarray(rgb, np.int32)
    r, g, b = x[..., 0], x[..., 1], x[..., 2]
    mx, mn = np.maximum(np.maximum(r, g), b), np.minimum(np.minimum(r, g), b)
    grey = mx == mn
    cr = np.where(grey, 1, mx - mn).astype(F32)
    s = (cr / np.where(grey, 1, mx).astype(F32)).astype(F32)
    rc = ((mx - r).astype(F32) / cr).astype(F32)
    gc = ((mx - g).astype(F32) / cr).astype(F32)
    bc = ((mx - b).astype(F32) / cr).astype(F32)
    h = np.where(r == mx, (bc - gc).astype(F32).astype(F64),
                 np.where(g == mx, (F64(2.0) + rc.astype(F64)) - bc.astype(F64),
                          (F64(4.0) + gc.astype(F64)) - rc.astype(F64))).astype(F32)
    h = np.fmod(h.astype(F64) / F64(6.0) + F64(1.0), F64(1.0)).astype(F32)
    hh = np.clip((h.astype(F64) * F64(255.0)).astype(np.int64), 0, 255)
    ss = np.clip((s.astype(F64) * F64(255.0)).astype(np.int64), 0, 255)
    out = np.empty(x.shape, np.uint8)
    out[..., 0] = np.where(grey, 0, hh)
    out[..., 1] = np.where(grey, 0, ss)
    out[..., 2] = mx
    return out


def _round_half_away(x):
    return np.where(x >= 0, np.floor(x + F64(0.5)), np.ceil(x - F64(0.5)))


def hsv_to_rgb(hsv):
    """Pillow's HSV->RGB on (..., 3) uint8.  float64 a = H * 6.0 / 255.0, i = floor(a), f = fl32(a - i),
    fs = fl32(S / 255.0); p = round(V * (1.0 - fs)), q = round(V * (1.0 - fl32(fs * f))),
    t = round(V * (1.0 - fs * (1.0 - f))), all float64 but fs * f, round half away from zero, clipped; then the
    sector i % 6 picks (V, t, p), (q, V, p), (p, V, t), (p, q, V), (t, p, V), (V, p, q).  S = 0 gives (V, V, V)."""
    x = np.asarray(hsv, np.int32)
    h, s, v = x[..., 0], x[..., 1], x[..., 2]
    a = h.astype(F64) * F64(6.0) / F64(255.0)
    i = np.floor(a).astype(np.int64)
    f = (a - i.astype(F32).astype(F64)).astype(F32)
    fs = (s.astype(F64) / F64(255.0)).astype(F32)
    vd = v.astype(F64)
    p = _round_half_away(vd * (F64(1.0) - fs.astype(F64)))
    q = _round_half_away(vd * (F64(1.0) - (fs * f).astype(F32).astype(F64)))
    t = _round_half_away(vd * (F64(1.0) - fs.astype(F64) * (F64(1.0) - f.astype(F64))))
    p, q, t = (np.clip(c, 0, 255).astype(np.int64) for c in (p, q, t))
    v = v.astype(np.int64)
    sector = i % 6
    table = [(v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q)]
    out = np.empty(x.shape, np.uint8)
    for c in range(3):
        ch = np.select([sector == k for k in range(6)], [table[k][c] for k in range(6)])
        out[..., c] = np.where(s == 0, v, ch)
    return out


def adjust_hue(rgb, hb):
    """adjust_hue with the shift byte hb = hue_byte(hue_factor)."""
    hsv = rgb_to_hsv(rgb)
    hsv[..., 0] = (hsv[..., 0].astype(np.int32) + int(hb)) & 255
    return hsv_to_rgb(hsv)


def apply_op(img, op, factors, hb):
    """One ColorJitter op on an (H, W, 3) uint8 image: op in BRIGHTNESS .. HUE, factors = (b, c, s)."""
    if op == BRIGHTNESS:
        return blend(0, img, factors[0])
    if op == CONTRAST:
        m = contrast_mean(int(rgb_to_l(img).astype(np.int64).sum()), img.shape[0] * img.shape[1])
        return blend(m, img, factors[1])
    if op == SATURATION:
        return blend(rgb_to_l(img)[..., None], img, factors[2])
    if op == HUE:
        return adjust_hue(img, hb)
    raise ValueError(f'unknown op {op}')


def jitter(img, order, factors, hue_factor):
    """ColorJitter.forward on an (H, W, 3) uint8 image given get_params' draws: order = fn_idx, factors = (b, c, s);
    an op whose factor is None is skipped."""
    out = np.asarray(img, np.uint8)
    present = list(factors) + [hue_factor]
    for op in order:
        if present[int(op)] is not None:
            out = apply_op(out, int(op), factors, hue_byte(hue_factor) if int(op) == HUE else 0)
    return out
