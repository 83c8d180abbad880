"""Restatement of the self-supervised loss (test infrastructure; DESIGN.md section 9.1).

`census` is the NumPy float32 census transform that the CUDA kernel (tf_raft_b200/csrc/unsup.cuh, census_kernel) must
match bit for bit: every operation is one float32 NumPy operation in the kernel's order.

`loss` / `direction_terms` restate the loss in float64 torch, differentiable with torch.autograd; `direction_closed_form`
restates one direction and its gradient in plain NumPy float64, chunk by chunk, at any size (no autograd graph):
  * mask m = not occluded (oracle/occlusion_np.py on the float32 final predictions) and the pixel at least 3 px from
    every border (its 7x7 census window inside the frame);
  * for prediction i, the landing p = (x, y) + F_i is taken in float32, as the kernel takes it, to decide the corners
    (x0 = floor(px), x1 = min(x0 + 1, W - 1)) and whether p lies in the closed frame; the weights ax = px - x0 are
    float64 with px = x + F_i, so floor carries no gradient and ax has gradient 1.  A landing outside the frame samples
    at (0, 0) instead and its penalty is replaced by 0, so it carries no gradient and no NaN;
  * D = sum_c d^2 / (0.1 + d^2), d = C_target - sampled C_source; rho = (D + 0.01)^0.4;
    L_c = sum_i gamma^(n-1-i) sum_x m rho / N, N = max(sum_x m, 1) unless a normaliser `census_norm` is given (a
    data-parallel rank's max(C, 1) / R, C the mask count of the whole batch, R the number of equal shards);
  * L_s = sum_i gamma^(n-1-i) (S_h + S_v) / 2, S_h / S_v the means over horizontal / vertical pairs of
    exp(-lambda mean_c |I_c(x') - I_c(x)| / 255) (|dFx| + |dFy|) / 2;
  * L = census_weight (L_c,fw + L_c,bw) / 2 + smoothness_weight (L_s,fw + L_s,bw) / 2.
"""
import numpy as np
import torch

from . import occlusion_np

F32 = np.float32
OFFSETS = [(dy, dx) for dy in range(-3, 4) for dx in range(-3, 4) if (dy, dx) != (0, 0)]


def grey(images):
    """(B, H, W, 3) float32 -> (B, H, W) float32: (0.2989 R + 0.5870 G + 0.1140 B) / 255 in that order."""
    im = np.asarray(images, dtype=F32)
    return (F32(0.2989) * im[..., 0] + F32(0.5870) * im[..., 1] + F32(0.1140) * im[..., 2]) / F32(255)


def census(images):
    """(B, H, W, 3) float32 in 0..255 -> (B, H, W, 48) float32."""
    g = grey(images)
    b, h, w = g.shape
    pad = np.zeros((b, h + 6, w + 6), dtype=F32)
    pad[:, 3:3 + h, 3:3 + w] = g
    out = np.empty((b, h, w, 48), dtype=F32)
    with np.errstate(invalid='ignore'):
        for k, (dy, dx) in enumerate(OFFSETS):
            t = pad[:, 3 + dy:3 + dy + h, 3 + dx:3 + dx + w] - g
            out[..., k] = t / np.sqrt(F32(0.81) + t * t)
    assert out.dtype == F32
    return out


def border_mask(b, h, w):
    m = np.zeros((b, h, w), dtype=bool)
    m[:, 3:h - 3, 3:w - 3] = True
    return m


def _t(a):
    return a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))


def sample(census_s, flow):
    """Bilinear sample of census_s (B, H, W, C) float64 at (x, y) + flow (B, H, W, 2) float64 -> (values, inside)."""
    b, h, w, _ = census_s.shape
    f32 = flow.detach().to(torch.float32)
    gy, gx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing='ij')
    px32, py32 = gx.float() + f32[..., 0], gy.float() + f32[..., 1]
    inside = (px32 >= 0) & (px32 <= w - 1) & (py32 >= 0) & (py32 <= h - 1)
    px = torch.where(inside, gx.double() + flow[..., 0], torch.zeros((), dtype=flow.dtype))
    py = torch.where(inside, gy.double() + flow[..., 1], torch.zeros((), dtype=flow.dtype))
    x0 = torch.where(inside, torch.floor(px32), torch.zeros(())).long()
    y0 = torch.where(inside, torch.floor(py32), torch.zeros(())).long()
    x1, y1 = torch.clamp(x0 + 1, max=w - 1), torch.clamp(y0 + 1, max=h - 1)
    ax, ay = (px - x0.double())[..., None], (py - y0.double())[..., None]
    bx, by = 1 - ax, 1 - ay
    bi = torch.arange(b)[:, None, None]
    c00, c01, c10, c11 = census_s[bi, y0, x0], census_s[bi, y0, x1], census_s[bi, y1, x0], census_s[bi, y1, x1]
    return by * (bx * c00 + ax * c01) + ay * (bx * c10 + ax * c11), inside


def distance(census_t, census_s, flow):
    """D (B, H, W) and the in-frame mask of one prediction."""
    s, inside = sample(census_s, flow)
    d = census_t - s
    return (d * d / (0.1 + d * d)).sum(-1), inside


def smoothness(image_t, flow, edge_weight):
    """(S_h + S_v) / 2 of one prediction."""
    def term(di, df):
        wgt = torch.exp(-edge_weight * di.abs().mean(-1) / 255.0)
        return (wgt * (df[..., 0].abs() + df[..., 1].abs()) / 2).mean()
    s_h = term(image_t[:, :, 1:] - image_t[:, :, :-1], flow[:, :, 1:] - flow[:, :, :-1])
    s_v = term(image_t[:, 1:] - image_t[:, :-1], flow[:, 1:] - flow[:, :-1])
    return (s_h + s_v) / 2


def direction_terms(census_t, census_s, image_t, mask, flows, gamma=0.8, edge_weight=150.0, census_norm=None):
    """(L_c, L_s) of one direction.  census_* (B, H, W, 48), image_t (B, H, W, 3), mask (B, H, W) bool; flows: the n
    predictions (B, H, W, 2); census_norm: the census normaliser instead of max(sum m, 1).  Everything is taken to
    float64; gradients reach the flows only."""
    census_t, census_s = _t(census_t).double(), _t(census_s).double()
    image_t = _t(image_t).double()
    m = _t(mask).double()
    n = len(flows)
    norm = max(float(m.sum()), 1.0) if census_norm is None else float(census_norm)
    lc = ls = 0.0
    for i, f in enumerate(flows):
        f = f.double()
        D, inside = distance(census_t, census_s, f)
        rho = torch.where(inside, (D + 0.01) ** 0.4, torch.zeros((), dtype=D.dtype))
        g = gamma ** (n - 1 - i)
        lc = lc + g * (m * rho).sum() / norm
        ls = ls + g * smoothness(image_t, f, edge_weight)
    return lc, ls


def _sgn(u):
    """d|u|/du as torch's abs backward: 0 at 0 and at NaN."""
    return np.where(u > 0, 1.0, np.where(u < 0, -1.0, 0.0))


def direction_closed_form(census_t, census_s, image_t, mask, flows, census_weight=1.0, smoothness_weight=0.5,
                          edge_weight=150.0, gamma=0.8, census_norm=None, pairs=None, chunk=1 << 15):
    """One direction in closed form: (L_c, L_s, mask count, grads), grads[i] (B, H, W, 2) float64 = d share / d F_i of
    the direction's share = census_weight / 2 L_c + smoothness_weight / 2 L_s.  Arguments as `direction_terms` (NumPy
    arrays or CPU tensors; the flows float32 or float64), under the same rules: landing, corners and in-frame test in
    float32, weights ax = (x + F_x) - x0 in float64 with gradient 1, d|u|/du = 0 at 0 and at NaN, a landing outside the
    frame contributes 0, edge weights in float64.  The census term visits masked pixels only, `chunk` at a time, so
    memory stays bounded at any size; the census features are taken to be finite (unmasked pixels then contribute
    exactly 0, as m * rho does in autograd).  The smoothness term runs per row band of at least `chunk` pixels, each
    band with a one-row halo below it.  pairs = (n_h, n_v): the numbers of horizontal and vertical pairs the smoothness
    means divide by, when the arrays are a band of a larger frame (default: those of the given shape)."""
    def arr(a, dt):
        return np.asarray(a.detach().cpu() if isinstance(a, torch.Tensor) else a, dtype=dt)
    ct = arr(census_t, F32).reshape(-1, 48)
    cs = arr(census_s, F32).reshape(-1, 48)
    img = arr(image_t, np.float64)
    mask = arr(mask, bool)
    flows = [arr(f, np.float64) for f in flows]
    b, h, w = mask.shape
    n = len(flows)
    count = int(mask.sum())
    norm = max(float(count), 1.0) if census_norm is None else float(census_norm)
    wgt = [gamma ** (n - 1 - i) for i in range(n)]
    grads = [np.zeros((b, h, w, 2)) for _ in range(n)]
    census_sum = [0.0] * n
    # census: every masked pixel, `chunk` at a time
    bi, yy, xx = np.nonzero(mask)
    for c0 in range(0, count, chunk):
        cb, cy, cx = bi[c0:c0 + chunk], yy[c0:c0 + chunk], xx[c0:c0 + chunk]
        tgt = ct[(cb * h + cy) * w + cx].astype(np.float64)
        for i, f in enumerate(flows):
            f64 = f[cb, cy, cx]
            f32 = f64.astype(F32)
            with np.errstate(invalid='ignore', over='ignore'):
                px32, py32 = cx.astype(F32) + f32[:, 0], cy.astype(F32) + f32[:, 1]
                ins = np.nonzero((px32 >= 0) & (px32 <= F32(w - 1)) & (py32 >= 0) & (py32 <= F32(h - 1)))[0]
            x0, y0 = np.floor(px32[ins]).astype(np.int64), np.floor(py32[ins]).astype(np.int64)
            x1, y1 = np.minimum(x0 + 1, w - 1), np.minimum(y0 + 1, h - 1)
            ax = ((cx[ins] + f64[ins, 0]) - x0)[:, None]
            ay = ((cy[ins] + f64[ins, 1]) - y0)[:, None]
            bx, by = 1 - ax, 1 - ay
            base = cb[ins] * h
            c00, c01 = cs[(base + y0) * w + x0], cs[(base + y0) * w + x1]
            c10, c11 = cs[(base + y1) * w + x0], cs[(base + y1) * w + x1]
            c00, c01, c10, c11 = (c.astype(np.float64) for c in (c00, c01, c10, c11))
            top, bot = bx * c00 + ax * c01, bx * c10 + ax * c11
            d = tgt[ins] - (by * top + ay * bot)
            e = 0.1 + d * d
            D = (d * d / e).sum(-1)
            q = 0.2 * d / (e * e)                                             # dD / dd
            gx = -(q * (by * (c01 - c00) + ay * (c11 - c10))).sum(-1)       # dD / dF_x
            gy = -(q * (bot - top)).sum(-1)
            census_sum[i] += float(((D + 0.01) ** 0.4).sum())
            k = 0.5 * census_weight * wgt[i] / norm * 0.4 * (D + 0.01) ** -0.6
            grads[i][cb[ins], cy[ins], cx[ins]] += np.stack([k * gx, k * gy], -1)
    # smoothness: row bands [r0, r1), the vertical pairs (y, y + 1) of y in the band, so the halo is row r1
    n_h, n_v = (b * h * (w - 1), b * (h - 1) * w) if pairs is None else pairs
    s_h, s_v = [0.0] * n, [0.0] * n
    rows = max(1, chunk // (b * w))
    for r0 in range(0, h, rows):
        r1 = min(h, r0 + rows)
        band = img[:, r0:min(h, r1 + 1)]
        wh = np.exp(-edge_weight * np.abs(band[:, :r1 - r0, 1:] - band[:, :r1 - r0, :-1]).mean(-1) / 255.0)
        wv = np.exp(-edge_weight * np.abs(band[:, 1:] - band[:, :-1]).mean(-1) / 255.0)
        for i, f in enumerate(flows):
            fb = f[:, r0:min(h, r1 + 1)]
            g = grads[i][:, r0:min(h, r1 + 1)]
            dh = fb[:, :r1 - r0, 1:] - fb[:, :r1 - r0, :-1]
            dv = fb[:, 1:] - fb[:, :-1]
            with np.errstate(invalid='ignore'):
                s_h[i] += float((wh * (np.abs(dh[..., 0]) + np.abs(dh[..., 1])) / 2).sum())
                s_v[i] += float((wv * (np.abs(dv[..., 0]) + np.abs(dv[..., 1])) / 2).sum())
            th = (smoothness_weight * wgt[i] / (8 * n_h)) * wh[..., None] * _sgn(dh)
            tv = (smoothness_weight * wgt[i] / (8 * n_v)) * wv[..., None] * _sgn(dv)
            g[:, :r1 - r0, 1:] += th
            g[:, :r1 - r0, :-1] -= th
            g[:, 1:] += tv
            g[:, :-1] -= tv
    lc = sum(wgt[i] * census_sum[i] for i in range(n)) / norm
    ls = sum(wgt[i] * (s_h[i] / n_h + s_v[i] / n_v) / 2 for i in range(n))
    return lc, ls, count, grads


def loss(image1, image2, preds_fw, preds_bw, census_weight=1.0, smoothness_weight=0.5, edge_weight=150.0, gamma=0.8,
         alpha1=0.01, alpha2=0.5, return_terms=False):
    """The whole loss: images (B, H, W, 3) in 0..255 (float32 arrays or tensors), preds_* lists of (B, H, W, 2)
    float tensors (may require grad)."""
    im1, im2 = (np.asarray(_t(im).detach().cpu(), dtype=F32) for im in (image1, image2))
    c1, c2 = census(im1), census(im2)
    occ_fw, occ_bw = occlusion_np.fb_occlusion(preds_fw[-1].detach().float().cpu().numpy(),
                                               preds_bw[-1].detach().float().cpu().numpy(), alpha1, alpha2)
    b, h, w, _ = im1.shape
    border = border_mask(b, h, w)
    fw = direction_terms(c1, c2, im1, border & ~occ_fw, preds_fw, gamma, edge_weight)
    bw = direction_terms(c2, c1, im2, border & ~occ_bw, preds_bw, gamma, edge_weight)
    total = census_weight * (fw[0] + bw[0]) / 2 + smoothness_weight * (fw[1] + bw[1]) / 2
    return (total, fw, bw) if return_terms else total
