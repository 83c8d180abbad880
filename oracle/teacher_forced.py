"""Teacher-forced float64 training references (test infrastructure; the product never imports this).

A float64 restatement of the training step parts from the fp32 GPU step after a few of RAFT's iterations: the two
trajectories of `coords1` drift apart, and the tf-raft sampler takes floor and ceil of every sampling position, so where
a position crosses an integer the coordinate gradient jumps.  Teacher forcing removes that cause.  The reference runs
with the GPU's own fp32 sampling positions as its values and lets the gradient flow through its own float64
coordinates; every floor, ceil and clip gate then agrees exactly with the kernel's, and what is left between the two is
rounding.  Everything else -- encoders, BatchNorm batch statistics, the GRU, convex upsampling, the loss -- runs free in
float64.

- `tf_positions`: the per-level, per-tap float32 positions of tf_raft_b200/csrc/train.cuh and lookup.cuh,
  u = fl32(fl32(c * 2^-l) + (a - r)).  `fl32(c * 2^-l + k)` in one rounding is not the same: a sum that crosses into the
  next binade can round onto an integer (c = 3 - 2^-22, k = 4 gives 7.0), where the kernel sees a zero-weight corner and
  a zero slope.
- `tf_retrieve`: oracle.raft_torch.CorrBlock.retrieve sampled at those positions, pos = exact + (u - exact).detach():
  the GPU's values, the identity as gradient.
- `grid_positions` / `grid_lookup`: the same for RAFT(conventions='pytorch'): ATen's grid_sample normalise and
  unnormalise in float32 as oracle/raft_pytorch._axis states them, then a float64 zero-padded bilinear sample at those
  pixel positions.  RAFT detaches the coordinates, so only the weights and the corners need to agree.
- `teacher_forced(recorded)`: a context in which oracle.raft_torch.forward samples every iteration's lookup at the
  next of the recorded fp32 coordinates (one (B, h, w, 2) tensor per iteration, in order).
"""
import contextlib

import torch

from oracle import raft_torch as rt


def tf_positions(coords32, level, radius):
    """coords32 (..., 2) float32 -> (..., 2r+1, 2r+1, 2) float32 sampling positions of `level`, laid out as
    CorrBlock.retrieve lays out centroid + delta: [..., i, j] = (x + d_i, y + d_j), d = -r..r."""
    assert coords32.dtype == torch.float32
    d = torch.arange(-radius, radius + 1, dtype=torch.float32, device=coords32.device)
    c = coords32 * (2.0 ** -level)                       # fl32(c * 2^-l): one rounding (exact unless subnormal)
    ux = c[..., 0, None, None] + d[:, None]              # fl32(cx_l + (a - r)), tap a along the first axis
    uy = c[..., 1, None, None] + d[None, :]              # fl32(cy_l + (b - r)), tap b along the second
    return torch.stack(torch.broadcast_tensors(ux, uy), dim=-1)


def tf_retrieve(corr_block, coords, coords32):
    """CorrBlock.retrieve at the float32 positions implied by `coords32` (values) with the gradient of `coords`
    (float64, (B, h, w, 2)) flowing through them as the identity."""
    r = corr_block.radius
    bs, h, w, _ = coords.shape
    d = torch.arange(-r, r + 1, dtype=coords.dtype, device=coords.device)
    dy, dx = torch.meshgrid(d, d, indexing='ij')
    delta = torch.stack([dy, dx], dim=-1).reshape(1, 2 * r + 1, 2 * r + 1, 2)
    c32 = coords32.reshape(bs * h * w, 2)
    out = []
    for i in range(corr_block.num_levels):
        exact = coords.reshape(bs * h * w, 1, 1, 2) / 2 ** i + delta
        u = tf_positions(c32, i, r).to(coords.dtype)
        s = rt.bilinear_sampler(corr_block.corr_pyramid[i], exact + (u - exact).detach())
        out.append(s.reshape(bs, h, w, -1))
    return torch.cat(out, dim=-1)


@contextlib.contextmanager
def teacher_forced(recorded):
    """Within the context, oracle.raft_torch.forward's k-th lookup samples at the positions of recorded[k] (float32
    coordinates, as the GPU's lookup received them).  Every recorded entry must be used."""
    queue = list(recorded)
    used = [0]
    original = rt.CorrBlock.retrieve

    def retrieve(self, coords):
        k = used[0]
        used[0] += 1
        return tf_retrieve(self, coords, queue[k].to(coords.device))

    rt.CorrBlock.retrieve = retrieve
    try:
        yield
    finally:
        rt.CorrBlock.retrieve = original
    assert used[0] == len(queue), f'{len(queue)} recorded lookups, {used[0]} used'


def grid_positions(v32, n):
    """ATen's grid_sample (align_corners=True) unnormalised pixel position of RAFT's normalised coordinate, in float32
    as oracle/raft_pytorch._axis computes it: g = fl(fl(2 v) * fl(1 / (n-1))) - 1, ix = fl(fl(g + 1) / 2) * (n-1);
    non-finite or out-of-int-range positions become -100 (ATen CUDA's safe_downgrade_to_int_range)."""
    assert v32.dtype == torch.float32
    nm1 = torch.tensor(float(n - 1), dtype=torch.float32, device=v32.device)
    g = (2 * v32) * (1 / nm1) - 1
    ix = ((g + 1) / 2) * nm1
    ok = (ix >= -2.0 ** 31) & (ix <= 2.0 ** 31)
    return torch.where(ok, ix, torch.full_like(ix, -100.0))


def _sample_zero_padded(img, ix, iy):
    """img (M, H, W) of any dtype; ix, iy (M, K) pixel positions of that dtype -> (M, K): bilinear with corners
    floor / floor + 1 and zero outside the frame (grid_sample's zeros padding)."""
    m, hh, ww = img.shape
    x0, y0 = ix.floor(), iy.floor()
    x1, y1 = x0 + 1, y0 + 1
    flat = img.reshape(m, hh * ww)
    out = torch.zeros_like(ix)
    for yy, wy in ((y0, y1 - iy), (y1, iy - y0)):
        for xx, wx in ((x0, x1 - ix), (x1, ix - x0)):
            ok = (xx >= 0) & (xx <= ww - 1) & (yy >= 0) & (yy <= hh - 1)
            idx = torch.where(ok, yy * ww + xx, torch.zeros_like(xx)).long()
            out = out + torch.where(ok, wy * wx * torch.gather(flat, 1, idx), torch.zeros_like(ix))
    return out


def grid_lookup(pyr, coords32, radius=4):
    """RAFT's CorrBlock.__call__ (oracle/raft_pytorch.corr_lookup) at the library's float32 grid_sample positions:
    pyr [(B*h*w, 1, h_l, w_l)] of any dtype, coords32 (B, 2, h, w) float32 (detached, as RAFT's) -> (B, levels *
    (2r+1)^2, h, w) in the pyramid's dtype, channel l*(2r+1)^2 + a*(2r+1) + b at x offset a - r, y offset b - r."""
    b, _, h, w = coords32.shape
    c = coords32.permute(0, 2, 3, 1).reshape(b * h * w, 2)
    d = torch.arange(-radius, radius + 1, dtype=torch.float32, device=c.device)
    s = 2 * radius + 1
    out = []
    for l, p in enumerate(pyr):
        hl, wl = p.shape[-2:]
        cl = c * (2.0 ** -l)
        ix = grid_positions(cl[:, 0, None] + d, wl).to(p.dtype)          # (Q, s): x of tap a
        iy = grid_positions(cl[:, 1, None] + d, hl).to(p.dtype)          # (Q, s): y of tap b
        ixx = ix[:, :, None].expand(-1, s, s).reshape(b * h * w, s * s)
        iyy = iy[:, None, :].expand(-1, s, s).reshape(b * h * w, s * s)
        out.append(_sample_zero_padded(p[:, 0], ixx, iyy).reshape(b, h, w, s * s))
    return torch.cat(out, dim=-1).permute(0, 3, 1, 2)


# ----------------------------------------------------------------------------- the tf-raft training step
FROZEN = ('moving_mean', 'moving_variance')


def sequence_loss(preds, flow_gt, valid, gamma=0.8, max_flow=400):
    """tf_raft/losses.py:4-21 on (B, H, W, 2) predictions in their own dtype and device: valid pixels with
    |flow_gt| < max_flow, the gamma-weighted means of |pred - flow_gt| over B*H*W*2."""
    fg = torch.as_tensor(flow_gt).to(preds[0])
    va = torch.as_tensor(valid).to(preds[0].device, torch.bool)
    vm = (va & (torch.sqrt((fg ** 2).sum(-1)) < max_flow)).to(fg.dtype).unsqueeze(-1)
    n = len(preds)
    return sum(gamma ** (n - i - 1) * (vm * (p - fg).abs()).mean() for i, p in enumerate(preds))


def tf_step(params, image1, image2, flow_gt, valid, variant, recorded, device='cpu', dtype=torch.float64):
    """One tf-raft training step's loss and gradients, teacher-forced by `recorded` (one float32 (B, h, w, 2) tensor of
    lookup coordinates per iteration): oracle.raft_torch.forward(training=True) in `dtype` on `device`, torch.autograd.
    Returns (loss, [predictions], {trainable name: gradient}, {BatchNorm layer: (batch mean, biased variance, count)})
    with tensors detached on `device`."""
    leaves = {k: torch.as_tensor(v).to(device, dtype).requires_grad_(not k.endswith(FROZEN)) for k, v in params.items()}
    names = [k for k, v in leaves.items() if v.requires_grad]
    rec = {}
    im1 = torch.as_tensor(image1).to(device, torch.float32)
    im2 = torch.as_tensor(image2).to(device, torch.float32)
    with teacher_forced(recorded):
        preds = rt.forward(leaves, im1, im2, variant, len(recorded), training=True, dtype=dtype, bn_record=rec)
    loss = sequence_loss(preds, flow_gt, valid)
    grads = torch.autograd.grad(loss, [leaves[k] for k in names])
    return float(loss), [p.detach() for p in preds], dict(zip(names, grads)), rec
