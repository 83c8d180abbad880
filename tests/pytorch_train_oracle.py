"""The original PyTorch RAFT's training step, restated on PyTorch-CPU in its own layout (test infrastructure for
RAFT(conventions='pytorch') training), next to `oracle/raft_pytorch.py`'s inference restatement, whose pieces it reuses.

- `lookup_backward_emulated`: raft_b200_corr_lookup_backward_ex(..., RAFT_SAMPLER_GRID) in NumPy float32, in the
  order stated in include/raft_b200.h, for bit-exact kernel tests.
- `train_forward`: RAFT.forward in training mode -- `F.batch_norm(training=..., momentum=0.1)` for cnet, the
  per-iteration `coords1 = coords1.detach()` -- differentiable in any dtype; `sequence_loss` is RAFT's.
- `TorchStep`: the real torch optimiser around it -- `clip_grad_norm_`, `torch.optim.AdamW(foreach=False)` and
  `OneCycleLR(..., pct_start=0.05, cycle_momentum=False, anneal_strategy='linear')`, in float64.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import raft_pytorch as rp

F32 = np.float32


# ----------------------------------------------------------------------------- the library's lookup backward, emulated
def lookup_backward_emulated(coords, grad_out, grad_pyr, radius):
    """grad_pyr[l] (B*h*w, h_l, w_l) float32 accumulators (copied, not modified) + the scatter of grad_out (B, h, w,
    levels*(2r+1)^2) through the grid_sample taps at coords (B, h, w, 2) -> the new accumulators.  Per query, taps in
    ascending t = a*(2r+1) + b, corners 00, 01, 10, 11; each in-frame corner adds fl(fl(wy * wx) * go) to its cell."""
    c = coords.reshape(-1, 2).astype(F32)
    nq = c.shape[0]
    s = 2 * radius + 1
    go = grad_out.reshape(nq, -1).astype(F32)
    d = np.arange(-radius, radius + 1).astype(F32)
    q = np.arange(nq)
    out = []
    for l, g in enumerate(grad_pyr):
        g = g.astype(F32).copy()
        hl, wl = g.shape[1:]
        inv = F32(1.0 / 2 ** l)
        vx = ((c[:, 0] * inv)[:, None] + d[None]).astype(F32)
        vy = ((c[:, 1] * inv)[:, None] + d[None]).astype(F32)
        wxf, wxc, x0, x1 = rp._axis(vx, wl)
        wyf, wyc, y0, y1 = rp._axis(vy, hl)
        for a in range(s):
            for b in range(s):
                gt = go[:, l * s * s + a * s + b]
                for wy, yi in ((wyf[:, b], y0[:, b]), (wyc[:, b], y1[:, b])):
                    for wx, xi in ((wxf[:, a], x0[:, a]), (wxc[:, a], x1[:, a])):
                        ok = (yi >= 0) & (xi >= 0)
                        qq, yy, xx = q[ok], yi[ok], xi[ok]
                        with np.errstate(all='ignore'):            # inf - inf, NaN: as the kernel computes them
                            term = ((wy * wx).astype(F32) * gt).astype(F32)
                            g[qq, yy, xx] = (g[qq, yy, xx] + term[ok]).astype(F32)
        out.append(g)
    return out


# ----------------------------------------------------------------------------- RAFT's training forward
def _norm(sd, x, name, kind, bn):
    if kind == 'instance':                                 # nn.InstanceNorm2d(affine=False)
        return F.instance_norm(x, eps=1e-5)
    return F.batch_norm(x, sd[name + '.running_mean'], sd[name + '.running_var'], sd[name + '.weight'],
                        sd[name + '.bias'], training=bn == 'train', momentum=0.1, eps=1e-5)


def _encoder(sd, x, prefix, kind, bn):
    """rp.encoder with BatchNorm in training (bn='train': batch statistics, running statistics updated in place) or
    eval mode (bn='frozen', RAFT's freeze_bn)."""
    x = F.relu(_norm(sd, rp._conv(sd, x, prefix + '.conv1', 2), prefix + '.norm1', kind, bn))
    for li, (_, stride) in enumerate(rp.STAGES, start=1):
        for bi, s in enumerate((stride, 1)):
            p = f'{prefix}.layer{li}.{bi}'
            y = F.relu(_norm(sd, rp._conv(sd, x, p + '.conv1', s), p + '.norm1', kind, bn))
            y = F.relu(_norm(sd, rp._conv(sd, y, p + '.conv2'), p + '.norm2', kind, bn))
            if s != 1:
                x = _norm(sd, rp._conv(sd, x, p + '.downsample.0', s), p + '.downsample.1', kind, bn)
            x = F.relu(x + y)
    return rp._conv(sd, x, prefix + '.conv2')


def train_forward(sd, image1, image2, iters, bn='train', dtype=torch.float64, lookup=None):
    """RAFT.forward(iters) with model.train() (and freeze_bn() for bn='frozen') on a state dict `sd` in PyTorch layout
    without the `module.` prefix (tensors of `dtype`; leaves that require grad are differentiated).  The running
    statistics in `sd` are updated in place under bn='train'.  Returns the `iters` upsampled flows, (B, H, W, 2).
    Runs on the device of `sd` (images: NumPy or tensors).  `lookup(k, pyramid, coords1)` replaces the k-th
    iteration's CorrBlock.__call__ (teacher forcing, oracle/teacher_forced.py); None is RAFT's own."""
    dev = sd['fnet.conv1.weight'].device
    im1 = torch.as_tensor(image1).to(dev, dtype).permute(0, 3, 1, 2)
    im2 = torch.as_tensor(image2).to(dev, dtype).permute(0, 3, 1, 2)
    im1 = 2 * (im1 / 255.0) - 1.0
    im2 = 2 * (im2 / 255.0) - 1.0
    b = im1.shape[0]
    fmap = _encoder(sd, torch.cat([im1, im2]), 'fnet', 'instance', bn)
    pyr = rp.corr_pyramid(fmap[:b], fmap[b:])
    cnet = _encoder(sd, im1, 'cnet', 'batch', bn)
    net, inp = torch.tanh(cnet[:, :128]), torch.relu(cnet[:, 128:])
    _, _, h, w = fmap.shape
    coords0 = rp.coords_grid(b, h, w, dtype).to(dev)
    coords1 = coords0.clone()
    preds = []
    for k in range(iters):
        coords1 = coords1.detach()
        corr = rp.corr_lookup(pyr, coords1) if lookup is None else lookup(k, pyr, coords1)
        net, mask, delta = rp.update_block(sd, net, inp, corr, coords1 - coords0)
        coords1 = coords1 + delta
        preds.append(rp.upsample_flow(coords1 - coords0, mask).permute(0, 2, 3, 1))
    return preds


def sequence_loss(preds, flow_gt, valid, gamma=0.8, max_flow=400):
    """RAFT's sequence_loss on (B, H, W, 2) predictions: valid >= 0.5 and |flow_gt| < max_flow, mean over B*H*W*2."""
    fg = torch.as_tensor(flow_gt).to(preds[0])
    va = torch.as_tensor(valid).to(preds[0])
    vm = ((va >= 0.5) & (torch.sqrt((fg ** 2).sum(-1)) < max_flow)).to(fg.dtype).unsqueeze(-1)
    n = len(preds)
    return sum(gamma ** (n - i - 1) * (vm * (p - fg).abs()).mean() for i, p in enumerate(preds))


def trainable(key):
    """RAFT's parameters (the optimiser's list): every conv weight / bias and cnet BatchNorm weight / bias; norm3 is
    the same module as downsample.1, so only the latter is listed."""
    return key.endswith(('.weight', '.bias')) and '.norm3.' not in key


class TorchStep:
    """RAFT's optimiser set-up in float64 on `sd` (PyTorch layout, no `module.` prefix): AdamW(lr, wd, eps) over the
    trainable leaves, OneCycleLR(lr, total_steps, pct_start=0.05, cycle_momentum=False, anneal_strategy='linear'),
    clip_grad_norm_(clip) before every step."""

    def __init__(self, sd, lr, wd, total_steps, clip, eps=1e-8):
        self.sd = {k: (v.detach().clone().double().requires_grad_(trainable(k)) if v.is_floating_point() else v)
                   for k, v in sd.items()}
        self.names = [k for k in self.sd if trainable(k)]
        params = [self.sd[k] for k in self.names]
        self.opt = torch.optim.AdamW(params, lr=lr, weight_decay=wd, eps=eps, foreach=False)
        self.sched = torch.optim.lr_scheduler.OneCycleLR(self.opt, lr, total_steps, pct_start=0.05,
                                                         cycle_momentum=False, anneal_strategy='linear')
        self.clip = clip

    def step(self, image1, image2, flow_gt, valid, iters, bn, gamma=0.8):
        """One training step; returns (loss, {name: gradient before the clip}, global norm)."""
        self.opt.zero_grad()
        loss = sequence_loss(train_forward(self.sd, image1, image2, iters, bn), flow_gt, valid, gamma)
        loss.backward()
        grads = {k: self.sd[k].grad.detach().clone() for k in self.names}
        norm = float(torch.nn.utils.clip_grad_norm_([self.sd[k] for k in self.names], self.clip))
        self.opt.step()
        self.sched.step()
        return float(loss), grads, norm

    def slot(self, name):
        """Adam's {name: tensor} of slot 'exp_avg' or 'exp_avg_sq'."""
        return {k: self.opt.state[self.sd[k]][name] for k in self.names}

    def load(self, sd):
        """Set the trainable leaves to the values of `sd` (PyTorch layout): the next gradient is taken there, while
        Adam's moments, the step count and the schedule stay the optimiser's own."""
        with torch.no_grad():
            for k in self.names:
                self.sd[k].copy_(torch.as_tensor(np.asarray(sd[k])).double())
