"""NumPy float32 restatement of the forward-backward occlusion check (test infrastructure).

`fb_occlusion` is what the CUDA kernel (tf_raft_b200/csrc/video.cuh, fb_occlusion_kernel) must match bit for bit: every
operation below is one float32 NumPy operation, rounded on its own, in the kernel's order.  For direction fw of image
b, with F = flow_fw[b] and G = flow_bw[b] (direction bw swaps them), pixel (x, y):
  * p = (x + fx, y + fy); the pixel is occluded unless 0 <= px <= W-1 and 0 <= py <= H-1 (NaN compares false);
  * g = bilinear sample of G at p: x0 = floor(px), x1 = min(x0 + 1, W-1), ax = px - x0, bx = 1 - ax (y likewise),
    g = by*(bx*G[y0,x0] + ax*G[y0,x1]) + ay*(bx*G[y1,x0] + ax*G[y1,x1]) per component;
  * consistent iff lhs <= rhs with lhs = sx*sx + sy*sy (s = f + g) and
    rhs = alpha1*((fx*fx + fy*fy) + (gx*gx + gy*gy)) + alpha2; otherwise occluded, NaN included.
tests/test_bidirectional.py checks it against an fp64 formulation built on scipy.ndimage.map_coordinates.
"""
import numpy as np

F32 = np.float32


def _one_direction(F, G, alpha1, alpha2, return_terms):
    b, h, w, _ = F.shape
    gy, gx = np.meshgrid(np.arange(h, dtype=F32), np.arange(w, dtype=F32), indexing='ij')
    fx, fy = F[..., 0], F[..., 1]
    px, py = gx[None] + fx, gy[None] + fy
    with np.errstate(invalid='ignore', over='ignore'):
        inside = (px >= F32(0)) & (px <= F32(w - 1)) & (py >= F32(0)) & (py <= F32(h - 1))
        # outside pixels sample at (0, 0); their result is discarded
        px, py = np.where(inside, px, F32(0)), np.where(inside, py, F32(0))
        fx0, fy0 = np.floor(px), np.floor(py)
        x0, y0 = fx0.astype(np.int64), fy0.astype(np.int64)
        x1, y1 = np.minimum(x0 + 1, w - 1), np.minimum(y0 + 1, h - 1)
        ax = px - fx0
        bx = F32(1) - ax
        ay = py - fy0
        by = F32(1) - ay
        bi = np.arange(b)[:, None, None]
        g00, g01, g10, g11 = G[bi, y0, x0], G[bi, y0, x1], G[bi, y1, x0], G[bi, y1, x1]
        g = by[..., None] * (bx[..., None] * g00 + ax[..., None] * g01) + \
            ay[..., None] * (bx[..., None] * g10 + ax[..., None] * g11)
        gxs, gys = g[..., 0], g[..., 1]
        sx, sy = fx + gxs, fy + gys
        lhs = sx * sx + sy * sy
        rhs = F32(alpha1) * ((fx * fx + fy * fy) + (gxs * gxs + gys * gys)) + F32(alpha2)
        occ = ~(inside & (lhs <= rhs))
    assert g.dtype == F32 and lhs.dtype == F32 and rhs.dtype == F32
    return (occ, inside, lhs, rhs) if return_terms else occ


def fb_occlusion(flow_fw, flow_bw, alpha1=0.01, alpha2=0.5, return_terms=False):
    """(B, H, W, 2) float32 flows a->b and b->a -> (occ_fw, occ_bw), bool (B, H, W).  With return_terms, each
    direction is (occ, inside, lhs, rhs) instead, lhs and rhs being meaningful where inside is True."""
    flow_fw = np.ascontiguousarray(flow_fw, dtype=F32)
    flow_bw = np.ascontiguousarray(flow_bw, dtype=F32)
    assert flow_fw.shape == flow_bw.shape and flow_fw.ndim == 4 and flow_fw.shape[-1] == 2
    return (_one_direction(flow_fw, flow_bw, alpha1, alpha2, return_terms),
            _one_direction(flow_bw, flow_fw, alpha1, alpha2, return_terms))
