"""NumPy float32 emulations of the training step's two fixed-order backward kernels, bit for bit (test infrastructure;
the product never imports this).

- `lookup_backward`: raft_b200_corr_lookup_backward (tf_raft_b200/csrc/train.cuh, corr_lookup_bwd_kernel).  The pyramid
  gradient is emulated as the literal scatter in the stated order (ascending tap, then corner), so it also checks the
  kernel's gather: that every term of a cell is found and added in that order.
- `upflow8_backward`: raft_b200_upflow8_backward (tf_raft_b200/csrc/kernels.cuh, upflow8_bwd_kernel), the adjoint of
  F.interpolate(scale_factor=8, mode='bilinear', align_corners=False) with PyTorch's weights.

Every operation below is one float32 operation, rounded once, as the kernels do it with __fmul_rn / __fadd_rn /
__fsub_rn."""
import numpy as np

F32 = np.float32


def _axis(c, offset, n):
    """One axis of one tap for every query: u = c + offset, g = clip(u, 0, n-1) (fminf / fmaxf: NaN clips to 0),
    corners floor(g) / ceil(g) with weights w1 = ceil(g) - g / w0 = g - floor(g), and the clip's gradient gate."""
    with np.errstate(invalid='ignore'):
        u = c + F32(offset)
        g = np.fmin(np.fmax(u, F32(0)), F32(n - 1))
        f0, f1 = np.floor(g), np.ceil(g)
        return dict(i0=f0.astype(np.int64), i1=f1.astype(np.int64), w0=g - f0, w1=f1 - g, gate=(u >= 0) & (u <= F32(n - 1)))


def lookup_backward(pyr, coords, grad_out, radius, grad_coords=None, grad_pyr=None):
    """pyr: levels float32 arrays (nq, h_l, w_l[, 1]); coords (..., 2) float32 with nq queries; grad_out (..., C) with
    the first levels*(2r+1)^2 channels read.  grad_coords / grad_pyr: the accumulators on entry (zeros if None).
    Returns (grad_coords (nq, 2), [grad_pyr_l (nq, h_l, w_l)]) as float32."""
    levels = len(pyr)
    side = 2 * radius + 1
    ntap = side * side
    c = np.ascontiguousarray(coords, dtype=F32).reshape(-1, 2)
    nq = c.shape[0]
    go_all = np.ascontiguousarray(grad_out, dtype=F32).reshape(nq, -1)
    gc = np.zeros((nq, 2), F32) if grad_coords is None else np.array(grad_coords, dtype=F32).reshape(nq, 2)
    rows = np.arange(nq)
    out_pyr, G = [], []
    for l in range(levels):
        P = np.ascontiguousarray(pyr[l], dtype=F32)
        H, W = P.shape[1], P.shape[2]
        P = P.reshape(nq, H * W)
        gp = (np.zeros((nq, H * W), F32) if grad_pyr is None else
              np.array(grad_pyr[l], dtype=F32).reshape(nq, H * W))
        inv = F32(1.0 / (1 << l))
        cx, cy = c[:, 0] * inv, c[:, 1] * inv
        lanes = np.zeros((2, nq, 32), F32)                               # +0 start of every lane sum
        with np.errstate(invalid='ignore', over='ignore', under='ignore'):
            for t in range(ntap):
                a, b = divmod(t, side)
                go = go_all[:, l * ntap + t]
                X, Y = _axis(cx, a - radius, W), _axis(cy, b - radius, H)
                p00 = P[rows, Y['i0'] * W + X['i0']]
                p01 = P[rows, Y['i0'] * W + X['i1']]
                p10 = P[rows, Y['i1'] * W + X['i0']]
                p11 = P[rows, Y['i1'] * W + X['i1']]
                live = go != 0
                dgx = go * (Y['w1'] * (p01 - p00) + Y['w0'] * (p11 - p10))
                dgy = go * (X['w1'] * (p10 - p00) + X['w0'] * (p11 - p01))
                # a skipped term adds nothing; adding +0 instead is the same, since a sum started at +0 is never -0
                lanes[0, :, t % 32] += np.where(live & X['gate'], dgx, F32(0))
                lanes[1, :, t % 32] += np.where(live & Y['gate'], dgy, F32(0))
                for yi, wy, xi, wx in ((Y['i0'], Y['w1'], X['i0'], X['w1']), (Y['i0'], Y['w1'], X['i1'], X['w0']),
                                       (Y['i1'], Y['w0'], X['i0'], X['w1']), (Y['i1'], Y['w0'], X['i1'], X['w0'])):
                    coef = wy * wx
                    m = live & (coef != 0)
                    q = rows[m]
                    cell = yi[m] * W + xi[m]
                    gp[q, cell] = gp[q, cell] + coef[m] * go[m]
            idx = np.arange(32)
            for o in (16, 8, 4, 2, 1):
                lanes = lanes + lanes[:, :, idx ^ o]
        G.append((lanes[0, :, 0], lanes[1, :, 0], inv))
        out_pyr.append(gp.reshape(nq, H, W))
    with np.errstate(invalid='ignore', over='ignore'):
        for gx, gy, inv in G:
            gc[:, 0] = gc[:, 0] + gx * inv
            gc[:, 1] = gc[:, 1] + gy * inv
    return gc, out_pyr


def upflow8_axis(n):
    """PyTorch upsample_bilinear2d (align_corners=False, scale 1/8) for the 8n output coordinates of an axis of n input
    cells: (i0, i1, l0, l1) arrays."""
    X = np.arange(8 * n, dtype=F32)
    src = np.maximum(F32(0.125) * (X + F32(0.5)) - F32(0.5), F32(0))
    i0 = src.astype(np.int64)
    i1 = i0 + (i0 < n - 1)
    l1 = src - i0.astype(F32)
    return i0, i1, F32(1) - l1, l1


def upflow8_backward(grad_up):
    """grad_up (B, 8h, 8w, 2) float32 -> grad_flow (B, h, w, 2) float32: each cell +0 plus its terms
    fl(fl(ly * lx) * g), in ascending output pixel (row-major) and then corner 00, 01, 10, 11, zero weights included."""
    g = np.ascontiguousarray(grad_up, dtype=F32)
    B, H, W, _ = g.shape
    h, w = H // 8, W // 8
    iy0, iy1, ly0, ly1 = upflow8_axis(h)
    ix0, ix1, lx0, lx1 = upflow8_axis(w)
    out = np.zeros((B, h, w, 2), F32)
    ys, xs = np.arange(h), np.arange(w)
    hits = 0
    with np.errstate(invalid='ignore', over='ignore'):
        # a gather over every cell at once: output rows Y = 8y - 8 + dY, dY ascending, hold every row whose corners can
        # land on row y (checked below: every corner of every output pixel is counted once)
        for dY in range(20):
            Y = 8 * ys - 8 + dY
            okY = (Y >= 0) & (Y < H)
            Yc = np.clip(Y, 0, H - 1)
            for dX in range(20):
                X = 8 * xs - 8 + dX
                okX = (X >= 0) & (X < W)
                Xc = np.clip(X, 0, W - 1)
                gv = g[:, Yc[:, None], Xc[None, :], :]
                for iy, ly in ((iy0, ly0), (iy1, ly1)):
                    for ix, lx in ((ix0, lx0), (ix1, lx1)):
                        hit = (okY & (iy[Yc] == ys))[:, None] & (okX & (ix[Xc] == xs))[None, :]
                        coef = ly[Yc][:, None] * lx[Xc][None, :]
                        out = np.where(hit[None, :, :, None], out + coef[None, :, :, None] * gv, out)
                        hits += int(hit.sum())
    assert hits == 4 * H * W, 'the 20 x 20 window missed a corner'
    return out
