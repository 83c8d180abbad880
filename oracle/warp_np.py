"""NumPy restatement of flow warping and flow composition (test infrastructure).

`warp` and `compose_flow` with dtype=float32 are what the CUDA kernels (tf_raft_b200/csrc/warp.cuh, warp_kernel and
compose_flow_kernel) must match bit for bit: every operation is one float32 NumPy operation, rounded on its own, in the
order include/raft_b200.h states.  For pixel (x, y) of image b with flow f:
  * p = (x + fx, y + fy) in float32; inside a (Hs, Ws) grid iff 0 <= px <= Ws-1 and 0 <= py <= Hs-1 (NaN compares false);
  * bilinear: x0 = floor(px), x1 = min(x0 + 1, Ws-1), ax = px - x0, bx = 1 - ax (y likewise),
    by*(bx*T[y0,x0] + ax*T[y0,x1]) + ay*(bx*T[y1,x0] + ax*T[y1,x1]);
  * nearest: xi = min(floor(px + 0.5), Ws-1), yi = min(floor(py + 0.5), Hs-1).
With dtype=float64 the landing p is still the float32 one (the kernel's positions) and everything after it is float64:
the accuracy reference for the blend (tests/test_warp_ref.py).  `track_forward` / `track_backward` spell out the
chaining of RAFT.track_video on given per-pair flows and masks.
"""
import numpy as np

F32 = np.float32


def _landing(flow, hs, ws):
    """flow (B, H, W, 2) -> float32 px, py (B, H, W) and the closed-frame test on an (hs, ws) grid."""
    flow = np.asarray(flow, F32)
    _, h, w, _ = flow.shape
    gy, gx = np.meshgrid(np.arange(h, dtype=F32), np.arange(w, dtype=F32), indexing='ij')
    with np.errstate(invalid='ignore', over='ignore'):
        px, py = gx[None] + flow[..., 0], gy[None] + flow[..., 1]
        inside = (px >= F32(0)) & (px <= F32(ws - 1)) & (py >= F32(0)) & (py <= F32(hs - 1))
    # outside pixels sample at (0, 0); their result is discarded
    return np.where(inside, px, F32(0)), np.where(inside, py, F32(0)), inside


def _bilinear(T, px, py, dtype):
    """Bilinear sample of T (B, Hs, Ws, C) at inside landings px, py (B, H, W) -> (B, H, W, C) in dtype."""
    _, hs, ws, _ = T.shape
    T = T.astype(dtype)
    fx0, fy0 = np.floor(px), np.floor(py)
    x0, y0 = fx0.astype(np.int64), fy0.astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, ws - 1), np.minimum(y0 + 1, hs - 1)
    one = dtype(1)
    ax = (px.astype(dtype) - fx0.astype(dtype))[..., None]
    ay = (py.astype(dtype) - fy0.astype(dtype))[..., None]
    bx, by = one - ax, one - ay
    bi = np.arange(T.shape[0])[:, None, None]
    with np.errstate(invalid='ignore', over='ignore'):
        out = by * (bx * T[bi, y0, x0] + ax * T[bi, y0, x1]) + ay * (bx * T[bi, y1, x0] + ax * T[bi, y1, x1])
    assert out.dtype == dtype
    return out


def bilinear_weight_sum(T, flow):
    """sum over the four corners of |weight * texel| in float64 at the float32 landings: the scale of the accuracy
    bound.  (B, H, W, C); 0 where the landing is outside."""
    px, py, inside = _landing(flow, T.shape[1], T.shape[2])
    return np.where(inside[..., None], _bilinear(np.abs(np.asarray(T, np.float64)), px, py, np.float64), 0.0)


def _nearest_index(px, py, hs, ws):
    with np.errstate(invalid='ignore'):
        xi = np.minimum(np.floor(px + F32(0.5)).astype(np.int64), ws - 1)
        yi = np.minimum(np.floor(py + F32(0.5)).astype(np.int64), hs - 1)
    return yi, xi


def warp(src, flow, mode='bilinear', fill=0, dtype=F32):
    """Backward warping.  src (B, Hs, Ws, C) float32 (or uint8 with mode='nearest'), flow (B, H, W, 2) float32 ->
    (out (B, H, W, C), occ bool (B, H, W)).  out is src's dtype (dtype for bilinear float), `fill` where occ."""
    src = np.asarray(src)
    b, hs, ws, _ = src.shape
    px, py, inside = _landing(flow, hs, ws)
    if mode == 'bilinear':
        assert src.dtype != np.uint8
        out = _bilinear(src, px, py, dtype)
    else:
        yi, xi = _nearest_index(px, py, hs, ws)
        out = src[np.arange(b)[:, None, None], yi, xi]
        if src.dtype != np.uint8:
            out = out.astype(dtype)
    out = np.where(inside[..., None], out, np.asarray(fill).astype(out.dtype))
    return out, ~inside


def compose_flow(f1, f2, occ1=None, occ2=None, dtype=F32):
    """out = f1 + bilinear(f2, x + f1); occ = occ1 | outside | occ2[nearest] | non-finite out; out = f1 where occ.
    (B, H, W, 2) flows, optional bool (B, H, W) masks -> (out, occ)."""
    f1 = np.asarray(f1, F32)
    b, h, w, _ = f1.shape
    px, py, inside = _landing(f1, h, w)
    with np.errstate(invalid='ignore', over='ignore'):
        s = f1.astype(dtype) + _bilinear(np.asarray(f2, F32), px, py, dtype)
    lost = ~inside | ~np.isfinite(s).all(-1)
    if occ1 is not None:
        lost |= np.asarray(occ1, bool)
    if occ2 is not None:
        yi, xi = _nearest_index(px, py, h, w)
        lost |= np.asarray(occ2, bool)[np.arange(b)[:, None, None], yi, xi] & inside
    return np.where(lost[..., None], f1.astype(dtype), s), lost


def track_forward(flows_fw, occs_fw):
    """Frame 0 -> t for t = 1 .. T-1 from the pairs' forward flows F_{t-1->t} and masks: a list of (flow, occ)."""
    acc, lost = np.asarray(flows_fw[0], F32), np.asarray(occs_fw[0], bool)
    out = [(acc, lost)]
    for f, o in zip(flows_fw[1:], occs_fw[1:]):
        acc, lost = compose_flow(acc, f, lost, o)
        out.append((acc, lost))
    return out


def track_backward(flows_bw, occs_bw):
    """Frame t -> 0 for t = 1 .. T-1 from the pairs' backward flows B_{t->t-1} and masks: a list of (flow, occ)."""
    acc, lost = np.asarray(flows_bw[0], F32), np.asarray(occs_bw[0], bool)
    out = [(acc, lost)]
    for f, o in zip(flows_bw[1:], occs_bw[1:]):
        acc, lost = compose_flow(f, acc, o, lost)
        out.append((acc, lost))
    return out
