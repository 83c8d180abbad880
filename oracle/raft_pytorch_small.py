"""The original PyTorch RAFT-small's inference (`raft-small.pth`, RAFT's `--small`), restated functionally on
PyTorch-CPU (test infrastructure), in the PyTorch layout of `oracle/raft_pytorch.py`, whose convolution, correlation
pyramid, grid_sample lookup and coordinate grid it shares: NCHW activations, OIHW weights, the original module paths
(`fnet.layer2.0.conv3.weight`, `cnet.layer3.0.downsample.0.weight`, ...).  `dtype=torch.float64` gives the reference
"truth".

`upflow8_emulated` is a NumPy float32 emulation of the library's align-corners upflow8
(raft_b200_upflow8_align_corners, include/raft_b200.h) in its stated operation order, for bit-exact kernel tests;
`upflow8_fp32_positions` interpolates in float64 at that kernel's (and ATen's) float32 source positions.
`synthetic_small_checkpoint` draws a seeded state dict shaped like `raft-small.pth`.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

from oracle.raft_pytorch import _conv, _sd, coords_grid, corr_lookup, corr_pyramid

SMALL_STAGES = ((32, 1), (64, 2), (96, 2))


def small_encoder(sd, x, prefix, kind, on_norm=None):
    """The original RAFT-small's SmallEncoder.forward (eval) on NCHW images already mapped to [-1, 1].  kind: 'instance'
    (nn.InstanceNorm2d(affine=False)) or 'none' (identity).  Bottleneck blocks: 1x1 -> 3x3 (stride) -> 1x1 at width
    planes / 4, each conv followed by its norm and ReLU, a 1x1 strided downsample (conv, norm4) when stride != 1, and
    relu(x + y).  on_norm(t), if given, sees the input of every instance norm."""
    def norm(t):
        if kind != 'instance':
            return t
        if on_norm is not None:
            on_norm(t)
        return F.instance_norm(t, eps=1e-5)

    x = F.relu(norm(_conv(sd, x, prefix + '.conv1', 2)))
    for li, (c, stride) in enumerate(SMALL_STAGES, start=1):
        for bi, s in enumerate((stride, 1)):
            p = f'{prefix}.layer{li}.{bi}'
            y = F.relu(norm(_conv(sd, x, p + '.conv1')))
            y = F.relu(norm(_conv(sd, y, p + '.conv2', s)))
            y = F.relu(norm(_conv(sd, y, p + '.conv3')))
            if s != 1:
                x = norm(_conv(sd, x, p + '.downsample.0', s))
            x = F.relu(x + y)
    return _conv(sd, x, prefix + '.conv2')


def small_update_block(sd, net, inp, corr, flow):
    """SmallUpdateBlock.forward -> (net, None, delta_flow): SmallMotionEncoder, ConvGRU(96, 146), FlowHead(96, 128)."""
    p = 'update_block.'
    cor = F.relu(_conv(sd, corr, p + 'encoder.convc1'))
    flo = F.relu(_conv(sd, flow, p + 'encoder.convf1'))
    flo = F.relu(_conv(sd, flo, p + 'encoder.convf2'))
    motion = torch.cat([F.relu(_conv(sd, torch.cat([cor, flo], 1), p + 'encoder.conv')), flow], 1)
    x = torch.cat([inp, motion], 1)
    hx = torch.cat([net, x], 1)
    z = torch.sigmoid(_conv(sd, hx, p + 'gru.convz'))
    r = torch.sigmoid(_conv(sd, hx, p + 'gru.convr'))
    q = torch.tanh(_conv(sd, torch.cat([r * net, x], 1), p + 'gru.convq'))
    net = (1 - z) * net + z * q
    return net, None, _conv(sd, F.relu(_conv(sd, net, p + 'flow_head.conv1')), p + 'flow_head.conv2')


def upflow8(flow):
    """RAFT-small's upflow8: 8 * F.interpolate(flow, size=(8h, 8w), mode='bilinear', align_corners=True), NCHW, in the
    flow's own dtype (float64 for the reference)."""
    n, _, h, w = flow.shape
    return 8 * F.interpolate(flow, size=(8 * h, 8 * w), mode='bilinear', align_corners=True)


def forward_small(state_dict, image1, image2, iters=12, flow_init=None, dtype=torch.float64):
    """RAFT(args.small).forward(test_mode=False) in eval: fnet SmallEncoder(128, 'instance'), cnet SmallEncoder(160,
    'none'), net / inp = tanh / relu of cnet split [96, 64], 4 levels at radius 3, upflow8 every iteration.  Arguments
    and result as `forward`."""
    sd = _sd(state_dict, dtype)
    im1 = torch.as_tensor(np.asarray(image1)).to(dtype).permute(0, 3, 1, 2)
    im2 = torch.as_tensor(np.asarray(image2)).to(dtype).permute(0, 3, 1, 2)
    im1 = 2 * (im1 / 255.0) - 1.0
    im2 = 2 * (im2 / 255.0) - 1.0
    b = im1.shape[0]
    with torch.no_grad():
        fmap = small_encoder(sd, torch.cat([im1, im2]), 'fnet', 'instance')
        pyr = corr_pyramid(fmap[:b], fmap[b:])
        cnet = small_encoder(sd, im1, 'cnet', 'none')
        net, inp = torch.tanh(cnet[:, :96]), torch.relu(cnet[:, 96:])
        _, _, h, w = fmap.shape
        coords0 = coords_grid(b, h, w, dtype)
        coords1 = coords0.clone()
        if flow_init is not None:
            coords1 = coords1 + torch.as_tensor(np.asarray(flow_init)).to(dtype).permute(0, 3, 1, 2)
        preds = []
        for _ in range(iters):
            corr = corr_lookup(pyr, coords1, radius=3)
            net, _, delta = small_update_block(sd, net, inp, corr, coords1 - coords0)
            coords1 = coords1 + delta
            preds.append(upflow8(coords1 - coords0).permute(0, 2, 3, 1).numpy())
        return preds, (coords1 - coords0).permute(0, 2, 3, 1).numpy()


def upflow8_emulated(flow):
    """raft_b200_upflow8_align_corners in NumPy float32, operation for operation (include/raft_b200.h): flow (B, h, w, 2)
    float32 -> (B, 8h, 8w, 2) float32."""
    f = np.float32
    flow = np.asarray(flow, np.float32)
    b, h, w, _ = flow.shape

    def axis(n):
        scale = f(f(n - 1) / f(8 * n - 1))
        src = (scale * np.arange(8 * n, dtype=np.float32)).astype(np.float32)
        i0 = src.astype(np.int64)                              # (int) truncation of a non-negative value
        i1 = i0 + (i0 < n - 1)
        l1 = (src - i0.astype(np.float32)).astype(np.float32)
        return i0, i1, (f(1) - l1).astype(np.float32), l1

    y0, y1, ly0, ly1 = axis(h)
    x0, x1, lx0, lx1 = axis(w)
    ly0, ly1 = ly0[None, :, None, None], ly1[None, :, None, None]
    lx0, lx1 = lx0[None, None, :, None], lx1[None, None, :, None]
    a, bb = flow[:, y0][:, :, x0], flow[:, y0][:, :, x1]
    c, d = flow[:, y1][:, :, x0], flow[:, y1][:, :, x1]
    with np.errstate(all='ignore'):
        top = (lx0 * a).astype(np.float32) + (lx1 * bb).astype(np.float32)
        bot = (lx0 * c).astype(np.float32) + (lx1 * d).astype(np.float32)
        val = (ly0 * top).astype(np.float32) + (ly1 * bot).astype(np.float32)
        return (f(8) * val).astype(np.float32)


def upflow8_fp32_positions(flow):
    """8 * bilinear align-corners upsampling of an NHWC flow (B, h, w, 2) in float64, at the float32 source positions
    ATen's kernel and `upflow8_emulated` use (scale = fl((n-1) / (8n-1)), src = fl(scale * X)): the exact interpolation
    of what the original RAFT-small's float32 upsampling samples."""
    flow = np.asarray(flow, np.float64)
    b, h, w, _ = flow.shape

    def axis(n):
        scale = np.float32(np.float32(n - 1) / np.float32(8 * n - 1))
        src = (scale * np.arange(8 * n, dtype=np.float32)).astype(np.float32).astype(np.float64)
        i0 = src.astype(np.int64)
        l1 = src - i0
        return i0, i0 + (i0 < n - 1), 1 - l1, l1

    y0, y1, ly0, ly1 = axis(h)
    x0, x1, lx0, lx1 = axis(w)
    ly0, ly1 = ly0[None, :, None, None], ly1[None, :, None, None]
    lx0, lx1 = lx0[None, None, :, None], lx1[None, None, :, None]
    top = lx0 * flow[:, y0][:, :, x0] + lx1 * flow[:, y0][:, :, x1]
    bot = lx0 * flow[:, y1][:, :, x0] + lx1 * flow[:, y1][:, :, x1]
    return 8 * (ly0 * top + ly1 * bot)


def _small_encoder_entries(prefix, out_dim):
    e = [(prefix + '.conv1', (32, 3, 7, 7))]
    cin = 32
    for li, (c, stride) in enumerate(SMALL_STAGES, start=1):
        for bi, s in enumerate((stride, 1)):
            p = f'{prefix}.layer{li}.{bi}'
            q = c // 4
            e += [(p + '.conv1', (q, cin, 1, 1)), (p + '.conv2', (q, q, 3, 3)), (p + '.conv3', (c, q, 1, 1))]
            if s != 1:
                e.append((p + '.downsample.0', (c, cin, 1, 1)))
            cin = c
    e.append((prefix + '.conv2', (out_dim, cin, 1, 1)))
    return e


def _small_update_entries():
    p = 'update_block.'
    return [(p + 'encoder.convc1', (96, 196, 1, 1)), (p + 'encoder.convf1', (64, 2, 7, 7)),
            (p + 'encoder.convf2', (32, 64, 3, 3)), (p + 'encoder.conv', (80, 128, 3, 3)),
            (p + 'gru.convz', (96, 242, 3, 3)), (p + 'gru.convr', (96, 242, 3, 3)), (p + 'gru.convq', (96, 242, 3, 3)),
            (p + 'flow_head.conv1', (128, 96, 3, 3)), (p + 'flow_head.conv2', (2, 128, 3, 3))]


def synthetic_small_checkpoint(seed=0, bias_scale=0.05):
    """A seeded state dict with the layout of the original `raft-small.pth`: `module.` prefix, OIHW float32 conv weights
    and biases, and nothing else (fnet's instance norms and cnet's 'none' norms hold no parameters or buffers).
    Kernels glorot-uniform, biases U(-bias_scale, bias_scale)."""
    rng = np.random.default_rng(seed)
    out = OrderedDict()
    entries = _small_encoder_entries('fnet', 128) + _small_encoder_entries('cnet', 160) + _small_update_entries()
    for name, shape in entries:
        o, i, kh, kw = shape
        lim = np.sqrt(6.0 / (kh * kw * (i + o)))
        out['module.' + name + '.weight'] = torch.as_tensor(rng.uniform(-lim, lim, shape), dtype=torch.float32)
        out['module.' + name + '.bias'] = torch.as_tensor(rng.uniform(-bias_scale, bias_scale, o), dtype=torch.float32)
    return out
