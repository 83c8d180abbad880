"""The original PyTorch RAFT's inference (basic model), restated functionally on PyTorch-CPU (test infrastructure).

Works on a state dict in PyTorch layout -- NCHW activations, OIHW weights, the original module paths
(`fnet.layer2.0.downsample.0.weight`, `cnet.norm1.running_var`, `update_block.mask.2.weight`, ...), the
`view(N, 1, 9, 8, 8, H, W)` mask layout -- so that it shares nothing with the loader that maps such a file onto this
project's parameters: a mistake in that mapping cannot be mirrored here.  Written independently of
`oracle/raft_torch.py` for every part where the two frameworks differ: `F.conv2d` with explicit symmetric padding,
`F.instance_norm` / `F.batch_norm` with eps = 1e-5, RAFT's `bilinear_sampler` (`F.grid_sample`, align_corners=True,
after 2 * x / (W - 1) - 1) and its convex upsampling.  `dtype=torch.float64` gives the reference "truth".

`lookup_emulated` is a NumPy float32 emulation of the library's grid_sample lookup (RAFT_SAMPLER_GRID,
include/raft_b200.h) in its stated operation order, for bit-exact kernel tests.  `synthetic_checkpoint` draws a seeded
PyTorch-layout checkpoint shaped like `raft-things.pth`.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

STAGES = ((64, 1), (96, 2), (128, 2))


def _sd(state_dict, dtype):
    return {(k[len('module.'):] if k.startswith('module.') else k): torch.as_tensor(v).to(dtype)
            for k, v in state_dict.items() if not k.endswith('num_batches_tracked')}


def _conv(sd, x, name, stride=1):
    w = sd[name + '.weight']
    return F.conv2d(x, w, sd[name + '.bias'], stride=stride, padding=((w.shape[2] - 1) // 2, (w.shape[3] - 1) // 2))


def _norm(sd, x, name, kind):
    if kind == 'instance':                                 # nn.InstanceNorm2d(affine=False)
        return F.instance_norm(x, eps=1e-5)
    return F.batch_norm(x, sd[name + '.running_mean'], sd[name + '.running_var'], sd[name + '.weight'],
                        sd[name + '.bias'], training=False, eps=1e-5)


def encoder(sd, x, prefix, kind):
    """BasicEncoder.forward (eval) on NCHW images already mapped to [-1, 1]."""
    x = F.relu(_norm(sd, _conv(sd, x, prefix + '.conv1', 2), prefix + '.norm1', kind))
    cin = 64
    for li, (c, stride) in enumerate(STAGES, start=1):
        for bi, s in enumerate((stride, 1)):
            p = f'{prefix}.layer{li}.{bi}'
            y = F.relu(_norm(sd, _conv(sd, x, p + '.conv1', s), p + '.norm1', kind))
            y = F.relu(_norm(sd, _conv(sd, y, p + '.conv2'), p + '.norm2', kind))
            if s != 1:                                     # ResidualBlock.downsample = (conv 1x1 s2, norm3)
                x = _norm(sd, _conv(sd, x, p + '.downsample.0', s), p + '.downsample.1', kind)
            x = F.relu(x + y)
            cin = c
    return _conv(sd, x, prefix + '.conv2')


def bilinear_sampler(img, coords):
    """RAFT's utils.bilinear_sampler: img (M, 1, H, W), coords (M, P, Q, 2) in pixels (x, y).

    As RAFT runs it, on CUDA: ATen's CUDA kernel sends a non-finite unnormalised coordinate to -100
    (safe_downgrade_to_int_range), so a level of height or width 1 (2x/0) and a NaN coordinate sample 0.  ATen's CPU
    kernel propagates the NaN instead, so such samples are set to 0 here."""
    H, W = img.shape[-2:]
    xgrid, ygrid = coords.split([1, 1], dim=-1)
    xgrid = 2 * xgrid / (W - 1) - 1
    ygrid = 2 * ygrid / (H - 1) - 1
    grid = torch.cat([xgrid, ygrid], dim=-1)
    ok = torch.isfinite(grid).all(dim=-1, keepdim=True)
    out = F.grid_sample(img, torch.where(ok, grid, torch.zeros_like(grid)), align_corners=True)
    return torch.where(ok.permute(0, 3, 1, 2), out, torch.zeros_like(out))


def corr_pyramid(fmap1, fmap2, levels=4):
    """CorrBlock.__init__: fmap (B, C, h, w) -> [(B*h*w, 1, h >> l, w >> l)]."""
    b, c, h, w = fmap1.shape
    corr = torch.matmul(fmap1.view(b, c, h * w).transpose(1, 2), fmap2.view(b, c, h * w)) / np.sqrt(c)
    pyr = [corr.reshape(b * h * w, 1, h, w)]
    for _ in range(levels - 1):
        pyr.append(F.avg_pool2d(pyr[-1], 2, stride=2))
    return pyr


def corr_lookup(pyr, coords, radius=4):
    """CorrBlock.__call__: coords (B, 2, h, w) -> (B, levels * (2r+1)^2, h, w)."""
    coords = coords.permute(0, 2, 3, 1)
    b, h, w, _ = coords.shape
    d = torch.linspace(-radius, radius, 2 * radius + 1, dtype=coords.dtype)
    delta = torch.stack(torch.meshgrid(d, d, indexing='ij'), dim=-1).view(1, 2 * radius + 1, 2 * radius + 1, 2)
    out = []
    for i, corr in enumerate(pyr):
        centroid = coords.reshape(b * h * w, 1, 1, 2) / 2 ** i
        out.append(bilinear_sampler(corr, centroid + delta).view(b, h, w, -1))
    return torch.cat(out, dim=-1).permute(0, 3, 1, 2)


def update_block(sd, net, inp, corr, flow):
    """BasicUpdateBlock.forward -> (net, mask, delta_flow)."""
    p = 'update_block.'
    cor = F.relu(_conv(sd, corr, p + 'encoder.convc1'))
    cor = F.relu(_conv(sd, cor, p + 'encoder.convc2'))
    flo = F.relu(_conv(sd, flow, p + 'encoder.convf1'))
    flo = F.relu(_conv(sd, flo, p + 'encoder.convf2'))
    motion = torch.cat([F.relu(_conv(sd, torch.cat([cor, flo], 1), p + 'encoder.conv')), flow], 1)
    x = torch.cat([inp, motion], 1)
    h = net
    for s in ('1', '2'):                                   # SepConvGRU: horizontal, then vertical
        hx = torch.cat([h, x], 1)
        z = torch.sigmoid(_conv(sd, hx, p + 'gru.convz' + s))
        r = torch.sigmoid(_conv(sd, hx, p + 'gru.convr' + s))
        q = torch.tanh(_conv(sd, torch.cat([r * h, x], 1), p + 'gru.convq' + s))
        h = (1 - z) * h + z * q
    delta = _conv(sd, F.relu(_conv(sd, h, p + 'flow_head.conv1')), p + 'flow_head.conv2')
    mask = .25 * _conv(sd, F.relu(_conv(sd, h, p + 'mask.0')), p + 'mask.2')
    return h, mask, delta


def upsample_flow(flow, mask):
    """RAFT.upsample_flow: (N, 2, H, W), (N, 576, H, W) -> (N, 2, 8H, 8W)."""
    n, _, h, w = flow.shape
    mask = torch.softmax(mask.view(n, 1, 9, 8, 8, h, w), dim=2)
    up = F.unfold(8 * flow, [3, 3], padding=1).view(n, 2, 9, 1, 1, h, w)
    up = torch.sum(mask * up, dim=2).permute(0, 1, 4, 2, 5, 3)
    return up.reshape(n, 2, 8 * h, 8 * w)


def coords_grid(b, h, w, dtype):
    y, x = torch.meshgrid(torch.arange(h, dtype=dtype), torch.arange(w, dtype=dtype), indexing='ij')
    return torch.stack([x, y])[None].repeat(b, 1, 1, 1)


def forward(state_dict, image1, image2, iters=12, flow_init=None, dtype=torch.float64):
    """RAFT.forward(test_mode=False) in eval.  image1, image2: (B, H, W, 3) 0..255 (NumPy or torch); flow_init:
    (B, H/8, W/8, 2) or None.  Returns (list of the `iters` upsampled flows (B, H, W, 2), final low-resolution flow
    (B, H/8, W/8, 2)) as NumPy arrays of `dtype`."""
    sd = _sd(state_dict, dtype)
    im1 = torch.as_tensor(np.asarray(image1)).to(dtype).permute(0, 3, 1, 2)
    im2 = torch.as_tensor(np.asarray(image2)).to(dtype).permute(0, 3, 1, 2)
    im1 = 2 * (im1 / 255.0) - 1.0
    im2 = 2 * (im2 / 255.0) - 1.0
    b = im1.shape[0]
    with torch.no_grad():
        fmap = encoder(sd, torch.cat([im1, im2]), 'fnet', 'instance')
        pyr = corr_pyramid(fmap[:b], fmap[b:])
        cnet = encoder(sd, im1, 'cnet', 'batch')
        net, inp = torch.tanh(cnet[:, :128]), torch.relu(cnet[:, 128:])
        _, _, h, w = fmap.shape
        coords0 = coords_grid(b, h, w, dtype)
        coords1 = coords0.clone()
        if flow_init is not None:
            coords1 = coords1 + torch.as_tensor(np.asarray(flow_init)).to(dtype).permute(0, 3, 1, 2)
        preds = []
        for _ in range(iters):
            corr = corr_lookup(pyr, coords1)
            net, mask, delta = update_block(sd, net, inp, corr, coords1 - coords0)
            coords1 = coords1 + delta
            preds.append(upsample_flow(coords1 - coords0, mask).permute(0, 2, 3, 1).numpy())
        return preds, (coords1 - coords0).permute(0, 2, 3, 1).numpy()


# ----------------------------------------------------------------------------- the library's lookup, emulated

def _axis(v, n):
    """Per-axis set-up of RAFT_SAMPLER_GRID in float32: (weight of x0, weight of x1, x0 or -1, x1 or -1)."""
    f = np.float32
    nm1 = f(n - 1)
    with np.errstate(all='ignore'):
        g = (f(2) * v) * (f(1) / nm1) - f(1)          # ATen CUDA: x / scalar is x * fl(1 / scalar)
        ix = ((g + f(1)) / f(2)) * nm1
    ix = np.where((ix >= -2.0 ** 31) & (ix <= 2.0 ** 31), ix, f(-100)).astype(np.float32)
    x0 = np.floor(ix)
    x1 = x0 + f(1)
    ok0 = (x0 >= 0) & (x0 <= nm1)
    ok1 = (x1 >= 0) & (x1 <= nm1)
    return x1 - ix, ix - x0, np.where(ok0, x0, -1).astype(np.int64), np.where(ok1, x1, -1).astype(np.int64)


def lookup_emulated(pyr, coords, radius):
    """raft_b200_corr_lookup_ex(..., RAFT_SAMPLER_GRID) in NumPy float32, operation for operation.
    pyr: [(B*h*w, h_l, w_l)] float32; coords (B, h, w, 2) float32 -> (B, h, w, levels * (2r+1)^2) float32."""
    f = np.float32
    b, h, w, _ = coords.shape
    c = coords.reshape(-1, 2).astype(np.float32)
    s = 2 * radius + 1
    d = np.arange(-radius, radius + 1).astype(np.float32)
    out = []
    q = np.arange(c.shape[0])[:, None, None]
    for l, img in enumerate(pyr):
        hl, wl = img.shape[1:]
        inv = f(1.0 / 2 ** l)
        vx = (c[:, 0] * inv)[:, None] + d[None]           # (Q, S): x of tap a
        vy = (c[:, 1] * inv)[:, None] + d[None]           # (Q, S): y of tap b
        wxf, wxc, x0, x1 = _axis(vx.astype(np.float32), wl)
        wyf, wyc, y0, y1 = _axis(vy.astype(np.float32), hl)
        acc = np.zeros((c.shape[0], s, s), np.float32)    # [q, a, b]
        for wy, yi in ((wyf, y0), (wyc, y1)):
            for wx, xi in ((wxf, x0), (wxc, x1)):
                ok = (yi[:, None, :] >= 0) & (xi[:, :, None] >= 0)
                v = img[q, np.maximum(yi, 0)[:, None, :], np.maximum(xi, 0)[:, :, None]]
                with np.errstate(all='ignore'):
                    t = (wy[:, None, :] * wx[:, :, None]) * v
                    acc = np.where(ok, acc + t, acc).astype(np.float32)
        out.append(acc.reshape(c.shape[0], s * s))
    return np.concatenate(out, axis=1).reshape(b, h, w, -1)


# ----------------------------------------------------------------------------- synthetic checkpoints

def _encoder_entries(prefix, kind, out_dim):
    e = [(prefix + '.conv1', 'conv', (64, 3, 7, 7))]
    if kind == 'batch':
        e.append((prefix + '.norm1', 'bn', 64))
    cin = 64
    for li, (c, stride) in enumerate(STAGES, start=1):
        for bi, s in enumerate((stride, 1)):
            p = f'{prefix}.layer{li}.{bi}'
            e += [(p + '.conv1', 'conv', (c, cin, 3, 3)), (p + '.conv2', 'conv', (c, c, 3, 3))]
            if kind == 'batch':
                e += [(p + '.norm1', 'bn', c), (p + '.norm2', 'bn', c)]
                if s != 1:
                    e.append((p + '.norm3', 'bn', c))
            if s != 1:
                e.append((p + '.downsample.0', 'conv', (c, cin, 1, 1)))
            cin = c
    e.append((prefix + '.conv2', 'conv', (out_dim, cin, 1, 1)))
    return e


def _update_entries():
    p = 'update_block.'
    e = [(p + 'encoder.convc1', (256, 324, 1, 1)), (p + 'encoder.convc2', (192, 256, 3, 3)),
         (p + 'encoder.convf1', (128, 2, 7, 7)), (p + 'encoder.convf2', (64, 128, 3, 3)),
         (p + 'encoder.conv', (126, 256, 3, 3))]
    e += [(f'{p}gru.conv{g}1', (128, 384, 1, 5)) for g in 'zrq']
    e += [(f'{p}gru.conv{g}2', (128, 384, 5, 1)) for g in 'zrq']
    e += [(p + 'flow_head.conv1', (256, 128, 3, 3)), (p + 'flow_head.conv2', (2, 256, 3, 3)),
          (p + 'mask.0', (256, 128, 3, 3)), (p + 'mask.2', (576, 256, 1, 1))]
    return [(n, 'conv', s) for n, s in e]


def synthetic_checkpoint(seed=0, bias_scale=0.05, norm_jitter=0.1):
    """A seeded state dict with the layout of the original RAFT's checkpoints (nn.DataParallel's `module.` prefix,
    OIHW float32 weights, BatchNorm `num_batches_tracked`, every cnet downsample norm stored twice as `norm3` and
    `downsample.1`).  Kernels glorot-uniform, biases U(-bias_scale, bias_scale), BatchNorm weight and running
    variance 1 + U(-j, j), bias and running mean U(-j, j)."""
    rng = np.random.default_rng(seed)
    sd = OrderedDict()
    entries = _encoder_entries('fnet', 'instance', 256) + _encoder_entries('cnet', 'batch', 256) + _update_entries()
    for name, kind, shape in entries:
        if kind == 'conv':
            o, i, kh, kw = shape
            lim = np.sqrt(6.0 / (kh * kw * (i + o)))
            sd[name + '.weight'] = rng.uniform(-lim, lim, shape)
            sd[name + '.bias'] = rng.uniform(-bias_scale, bias_scale, o)
        else:
            c = shape
            sd[name + '.weight'] = 1 + rng.uniform(-norm_jitter, norm_jitter, c)
            sd[name + '.bias'] = rng.uniform(-norm_jitter, norm_jitter, c)
            sd[name + '.running_mean'] = rng.uniform(-norm_jitter, norm_jitter, c)
            sd[name + '.running_var'] = 1 + rng.uniform(-norm_jitter, norm_jitter, c)
            sd[name + '.num_batches_tracked'] = np.array(1000, np.int64)
    out = OrderedDict()
    for k, v in sd.items():
        t = torch.as_tensor(v) if v.dtype == np.int64 else torch.as_tensor(v, dtype=torch.float32)
        out['module.' + k] = t
        if '.norm3.' in k:                                 # ResidualBlock registers norm3 again as downsample[1]
            out['module.' + k.replace('.norm3.', '.downsample.1.')] = t.clone()
    return out
