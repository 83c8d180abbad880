"""Restatement of the self-supervised loss (test infrastructure; DESIGN.md section 9.1).

`census` is the NumPy float32 census transform that the CUDA kernel (tf_raft_b200/csrc/unsup.cuh, census_kernel) must
match bit for bit: every operation is one float32 NumPy operation in the kernel's order.

`loss` / `direction_terms` restate the loss in float64 torch, differentiable with torch.autograd:
  * mask m = not occluded (oracle/occlusion_np.py on the float32 final predictions) and the pixel at least 3 px from
    every border (its 7x7 census window inside the frame);
  * for prediction i, the landing p = (x, y) + F_i is taken in float32, as the kernel takes it, to decide the corners
    (x0 = floor(px), x1 = min(x0 + 1, W - 1)) and whether p lies in the closed frame; the weights ax = px - x0 are
    float64 with px = x + F_i, so floor carries no gradient and ax has gradient 1.  A landing outside the frame samples
    at (0, 0) instead and its penalty is replaced by 0, so it carries no gradient and no NaN;
  * D = sum_c d^2 / (0.1 + d^2), d = C_target - sampled C_source; rho = (D + 0.01)^0.4;
    L_c = sum_i gamma^(n-1-i) sum_x m rho / max(sum_x m, 1);
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


def direction_terms(census_t, census_s, image_t, mask, flows, gamma=0.8, edge_weight=150.0):
    """(L_c, L_s) of one direction.  census_* (B, H, W, 48), image_t (B, H, W, 3), mask (B, H, W) bool; flows: the n
    predictions (B, H, W, 2).  Everything is taken to float64; gradients reach the flows only."""
    census_t, census_s = _t(census_t).double(), _t(census_s).double()
    image_t = _t(image_t).double()
    m = _t(mask).double()
    n = len(flows)
    lc = ls = 0.0
    for i, f in enumerate(flows):
        f = f.double()
        D, inside = distance(census_t, census_s, f)
        rho = torch.where(inside, (D + 0.01) ** 0.4, torch.zeros((), dtype=D.dtype))
        g = gamma ** (n - 1 - i)
        lc = lc + g * (m * rho).sum() / max(float(m.sum()), 1.0)
        ls = ls + g * smoothness(image_t, f, edge_weight)
    return lc, ls


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
