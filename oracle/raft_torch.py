"""PyTorch-CPU functional restatement of the reference forward (test infrastructure).

Follows tf_raft/model.py:10-109,173-226, tf_raft/layers/{corr,update,extractor}.py
op for op with TF semantics per SURVEY.md Appendix A, but with fast kernels
(`F.conv2d`, `torch.bmm`) so that full-size cases (448x512, 12 iterations) finish
in seconds.  It is the second, independent oracle: `tests/test_oracle_*.py` check it
against the literal NumPy restatement (`oracle.corr_np`, `oracle.tf_ops`).

All public tensors are NHWC float32 (NumPy or torch CPU), coords are (x, y).
`dtype=torch.float64` runs the same code in double as the error-budget "truth".
`quant=` (callable on tensors) is applied to every conv / matmul operand; the
precision study in DESIGN.md uses it to emulate TF32 / BF16 operand rounding.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


def _t(x, dtype=torch.float32):
    if isinstance(x, torch.Tensor):
        return x.to(dtype)
    return torch.from_numpy(np.ascontiguousarray(x)).to(dtype)


def _same_pads(n_in, k, s):
    n_out = -(-n_in // s)
    total = max((n_out - 1) * s + k - n_in, 0)
    return total // 2, total - total // 2


class Ops:
    """Conv / norm primitives on NCHW tensors bound to a parameter dict."""

    def __init__(self, params, dtype=torch.float32, quant=None, split=None, bn_record=None):
        self.dtype = dtype
        self.quant = quant
        self.split = split          # None | (xh_q, xl_q, wh_q, wl_q): emulate split-precision tensor-core passes
        # None | dict: every training-mode BatchNorm layer stores (batch mean, biased batch variance, count) under its
        # name, detached -- what oracle.train_ref.bn_moving_update advances the moving statistics with
        self.bn_record = bn_record
        self.p = {k: _t(v, dtype) for k, v in params.items()}
        self._wcache = {}

    def q(self, x):
        return x if self.quant is None else self.quant(x)

    def conv(self, x, name, stride=1, padding='same'):
        """keras Conv2D (HWIO kernel, cross-correlation, TF SAME padding incl. the asymmetric s=2 case)."""
        w = self._wcache.get(name)
        if w is None:
            w = self.q(self.p[name + '.kernel'].permute(3, 2, 0, 1).contiguous())
            self._wcache[name] = w
        kh, kw = w.shape[2], w.shape[3]
        if padding == 'same':
            pt, pb = _same_pads(x.shape[2], kh, stride)
            pl, pr = _same_pads(x.shape[3], kw, stride)
            if pt or pb or pl or pr:
                x = F.pad(x, (pl, pr, pt, pb))
        if self.split is not None:
            # three tensor-core passes on (hi, lo) operand splits: xh*wh + xl*wh + xh*wl, fp32 accumulate
            xh_q, xl_q, wh_q, wl_q = self.split
            w_raw = self.p[name + '.kernel'].permute(3, 2, 0, 1).contiguous()
            w_hi = wh_q(w_raw)
            w_lo = wl_q(w_raw - w_hi)
            x_hi = xh_q(x)
            x_lo = xl_q(x - x_hi)
            y = F.conv2d(x_hi, w_hi, self.p[name + '.bias'], stride=stride)
            return y + F.conv2d(x_lo, w_hi, None, stride=stride) + F.conv2d(x_hi, w_lo, None, stride=stride)
        return F.conv2d(self.q(x), w, self.p[name + '.bias'], stride=stride)

    def norm(self, x, name, norm_type, training):
        """extractor.py:6-16.  eps = 1e-3 for both tfa InstanceNormalization and keras BatchNormalization."""
        eps = 1e-3
        if norm_type is None:
            return x
        g = self.p[name + '.gamma'].view(1, -1, 1, 1)
        b = self.p[name + '.beta'].view(1, -1, 1, 1)
        if norm_type == 'instance':
            mean = x.mean(dim=(2, 3), keepdim=True)
            var = x.var(dim=(2, 3), unbiased=False, keepdim=True)
        elif norm_type == 'batch':
            if training:
                mean = x.mean(dim=(0, 2, 3), keepdim=True)
                var = x.var(dim=(0, 2, 3), unbiased=False, keepdim=True)
                if self.bn_record is not None:
                    self.bn_record[name] = (mean.detach().flatten(), var.detach().flatten(),
                                            x.shape[0] * x.shape[2] * x.shape[3])
            else:
                mean = self.p[name + '.moving_mean'].view(1, -1, 1, 1)
                var = self.p[name + '.moving_variance'].view(1, -1, 1, 1)
        else:
            raise ValueError(f'Invalid norm_type specified: {norm_type}')
        return (x - mean) * torch.rsqrt(var + eps) * g + b


# ----------------------------------------------------------------------------- extractor.py

def res_block(ops, x, prefix, norm_type, stride, training):
    """extractor.py:19-49."""
    fx = F.relu(ops.norm(ops.conv(x, prefix + '.conv1', stride), prefix + '.norm1', norm_type, training))
    fx = F.relu(ops.norm(ops.conv(fx, prefix + '.conv2', 1), prefix + '.norm2', norm_type, training))
    if stride != 1:
        x = ops.conv(x, prefix + '.downsample.0', stride, padding='valid')
        x = ops.norm(x, prefix + '.downsample.1', norm_type, training)
    return F.relu(x + fx)


def encoder(ops, x, prefix, norm_type, training):
    """BasicEncoder / SmallEncoder .call (extractor.py:113-130 / 158-175) on an NCHW tensor."""
    x = F.relu(ops.norm(ops.conv(x, prefix + '.conv1', 2), prefix + '.norm1', norm_type, training))
    for li, s in ((1, 1), (2, 2), (3, 2)):
        x = res_block(ops, x, f'{prefix}.layer{li}.0', norm_type, s, training)
        x = res_block(ops, x, f'{prefix}.layer{li}.1', norm_type, 1, training)
    return ops.conv(x, prefix + '.conv2', 1, padding='valid')


# ----------------------------------------------------------------------------- corr.py

def coords_grid(batch_size, height, width, dtype=torch.float32, device=None):
    """corr.py:72-90 -> (B, H, W, 2), (x, y)."""
    gy, gx = torch.meshgrid(torch.arange(height, dtype=dtype, device=device),
                            torch.arange(width, dtype=dtype, device=device), indexing='ij')
    return torch.stack([gx, gy], dim=-1)[None].repeat(batch_size, 1, 1, 1)


def bilinear_sampler(image, coords):
    """corr.py:28-69.  image (M, H, W, 1), coords (M, P, Q, 2) -> (M, P, Q, 1).  floor/ceil corners."""
    m, h, w, _ = image.shape
    gx = coords[..., 0].clamp(0, w - 1)
    gy = coords[..., 1].clamp(0, h - 1)
    gx0, gx1, gy0, gy1 = gx.floor(), gx.ceil(), gy.floor(), gy.ceil()
    img = image.reshape(m, h * w)

    def g(yy, xx):
        idx = (yy.long() * w + xx.long()).reshape(m, -1)
        return torch.gather(img, 1, idx).reshape(gx.shape)

    out = ((gy1 - gy) * (gx1 - gx) * g(gy0, gx0) + (gy1 - gy) * (gx - gx0) * g(gy0, gx1)
           + (gy - gy0) * (gx1 - gx) * g(gy1, gx0) + (gy - gy0) * (gx - gx0) * g(gy1, gx1))
    return out[..., None]


def upflow8(flow):
    """corr.py:93-96 on NHWC: 8 * bilinear resize with half-pixel centres."""
    x = flow.permute(0, 3, 1, 2)
    up = F.interpolate(x, scale_factor=8, mode='bilinear', align_corners=False)
    return 8 * up.permute(0, 2, 3, 1)


class CorrBlock:
    """corr.py:99-162 on NHWC torch tensors."""

    def __init__(self, fmap1, fmap2, num_levels=4, radius=4, quant=None):
        self.fmap1, self.fmap2 = fmap1, fmap2
        self.num_levels, self.radius = num_levels, radius
        self.quant = quant
        corr = self.correlation(fmap1, fmap2)
        bs, h1, w1, _, h2, w2 = corr.shape
        corr = corr.reshape(bs * h1 * w1, 1, h2, w2)
        self.corr_pyramid = [corr.permute(0, 2, 3, 1)]
        for _ in range(num_levels - 1):
            corr = F.avg_pool2d(corr, 2, 2)                       # VALID: floors odd dims
            self.corr_pyramid.append(corr.permute(0, 2, 3, 1))

    def retrieve(self, coords):
        r = self.radius
        bs, h, w, _ = coords.shape
        d = torch.arange(-r, r + 1, dtype=coords.dtype, device=coords.device)
        dy, dx = torch.meshgrid(d, d, indexing='ij')
        delta = torch.stack([dy, dx], dim=-1).reshape(1, 2 * r + 1, 2 * r + 1, 2)
        out = []
        for i in range(self.num_levels):
            centroid = coords.reshape(bs * h * w, 1, 1, 2) / 2 ** i
            s = bilinear_sampler(self.corr_pyramid[i], centroid + delta)
            out.append(s.reshape(bs, h, w, -1))
        return torch.cat(out, dim=-1)

    def correlation(self, fmap1, fmap2):
        bs, h, w, c = fmap1.shape
        q = (lambda t: t) if self.quant is None else self.quant
        f1 = q(fmap1.reshape(bs, h * w, c))
        f2 = q(fmap2.reshape(bs, h * w, c))
        corr = torch.bmm(f1, f2.transpose(1, 2)).reshape(bs, h, w, 1, h, w)
        return corr / math.sqrt(c) if fmap1.dtype == torch.float64 else corr / torch.sqrt(torch.tensor(float(c)))


# ----------------------------------------------------------------------------- update.py

def flow_head(ops, x, prefix):
    """update.py:5-14."""
    return ops.conv(F.relu(ops.conv(x, prefix + '.conv1')), prefix + '.conv2')


def conv_gru(ops, h, x, prefix):
    """update.py:17-35."""
    hx = torch.cat([h, x], dim=1)
    z = torch.sigmoid(ops.conv(hx, prefix + '.convz'))
    r = torch.sigmoid(ops.conv(hx, prefix + '.convr'))
    q = torch.tanh(ops.conv(torch.cat([r * h, x], dim=1), prefix + '.convq'))
    return (1 - z) * h + z * q


def sep_conv_gru(ops, h, x, prefix):
    """update.py:38-67: horizontal (1x5) pass then vertical (5x1) pass."""
    for s in ('1', '2'):
        hx = torch.cat([h, x], dim=1)
        z = torch.sigmoid(ops.conv(hx, prefix + '.convz' + s))
        r = torch.sigmoid(ops.conv(hx, prefix + '.convr' + s))
        q = torch.tanh(ops.conv(torch.cat([r * h, x], dim=1), prefix + '.convq' + s))
        h = (1 - z) * h + z * q
    return h


def basic_motion_encoder(ops, flow, corr, prefix):
    """update.py:88-106."""
    cor = F.relu(ops.conv(corr, prefix + '.convc1', padding='valid'))
    cor = F.relu(ops.conv(cor, prefix + '.convc2'))
    flo = F.relu(ops.conv(flow, prefix + '.convf1'))
    flo = F.relu(ops.conv(flo, prefix + '.convf2'))
    out = F.relu(ops.conv(torch.cat([cor, flo], dim=1), prefix + '.conv'))
    return torch.cat([out, flow], dim=1)


def small_motion_encoder(ops, flow, corr, prefix):
    """update.py:70-85."""
    cor = F.relu(ops.conv(corr, prefix + '.convc1'))
    flo = F.relu(ops.conv(flow, prefix + '.convf1'))
    flo = F.relu(ops.conv(flo, prefix + '.convf2'))
    out = F.relu(ops.conv(torch.cat([cor, flo], dim=1), prefix + '.conv'))
    return torch.cat([out, flow], dim=1)


def basic_update_block(ops, net, inp, corr, flow, prefix='update_block'):
    """update.py:143-153 on NCHW -> (net, 0.25*mask, delta_flow)."""
    motion = basic_motion_encoder(ops, flow, corr, prefix + '.encoder')
    x = torch.cat([inp, motion], dim=1)
    net = sep_conv_gru(ops, net, x, prefix + '.gru')
    delta = flow_head(ops, net, prefix + '.flow_head')
    mask = ops.conv(F.relu(ops.conv(net, prefix + '.mask.0')), prefix + '.mask.2', padding='valid')
    return net, 0.25 * mask, delta


def small_update_block(ops, net, inp, corr, flow, prefix='update_block'):
    """update.py:118-125 on NCHW -> (net, None, delta_flow)."""
    motion = small_motion_encoder(ops, flow, corr, prefix + '.encoder')
    x = torch.cat([inp, motion], dim=1)
    net = conv_gru(ops, net, x, prefix + '.gru')
    return net, None, flow_head(ops, net, prefix + '.flow_head')


# ----------------------------------------------------------------------------- model.py

def upsample_flow(flow, mask):
    """RAFT.upsample_flow (model.py:39-66) on NHWC: flow (B,h,w,2), mask (B,h,w,576) -> (B,8h,8w,2).

    mask channel = (by*8+bx)*9 + k, k = ky*3+kx over the zero-padded 3x3 neighbourhood of 8*flow.
    """
    bs, h, w, _ = flow.shape
    m = torch.softmax(mask.reshape(bs, h, w, 8, 8, 9, 1), dim=5)
    f = F.pad(8 * flow, (0, 0, 1, 1, 1, 1))
    patches = torch.stack([f[:, ky:ky + h, kx:kx + w, :] for ky in range(3) for kx in range(3)], dim=3)
    up = (m * patches.reshape(bs, h, w, 1, 1, 9, 2)).sum(dim=5)           # (B,h,w,8,8,2)
    return up.permute(0, 1, 3, 2, 4, 5).reshape(bs, 8 * h, 8 * w, 2)


VARIANTS = {
    'raft': dict(hidden=128, context=128, levels=4, radius=4, fnorm='instance', cnorm='batch'),
    'small': dict(hidden=96, context=64, levels=4, radius=3, fnorm='instance', cnorm=None),
}


def forward(params, image1, image2, variant='raft', iters=12, training=False,
            dtype=torch.float32, quant=None, split=None, return_intermediates=False, bn_record=None):
    """RAFT.call (model.py:68-109) / SmallRAFT.call (model.py:190-226).

    image1/2: (B, H, W, 3) in 0..255.  Returns the list of `iters` NHWC flow predictions
    (torch tensors); with return_intermediates also a dict of the tensors at the kernel
    boundaries (fmaps, net/inp, per-iteration corr/net/mask/delta/coords).  `bn_record` (a dict)
    receives the batch statistics of every training-mode BatchNorm layer (see Ops).
    """
    cfg = VARIANTS[variant]
    ops = Ops(params, dtype, quant, split, bn_record)
    x1 = _t(image1, dtype)
    x2 = _t(image2, dtype)
    bs, H, W, _ = x1.shape
    x1 = 2 * (x1 / 255.0) - 1.0                                             # model.py:70-71
    x2 = 2 * (x2 / 255.0) - 1.0
    both = torch.cat([x1, x2], dim=0).permute(0, 3, 1, 2)
    fm = encoder(ops, both, 'fnet', cfg['fnorm'], training).permute(0, 2, 3, 1)
    fmap1, fmap2 = fm[:bs].contiguous(), fm[bs:].contiguous()              # model.py:74
    corr_block = CorrBlock(fmap1, fmap2, cfg['levels'], cfg['radius'], quant)   # :77-79
    cnet = encoder(ops, x1.permute(0, 3, 1, 2), 'cnet', cfg['cnorm'], training)  # :82
    net = torch.tanh(cnet[:, :cfg['hidden']])                               # :84-86
    inp = F.relu(cnet[:, cfg['hidden']:])
    coords0 = coords_grid(bs, H // 8, W // 8, dtype, x1.device)             # :89, :32-37
    coords1 = coords0.clone()
    inter = dict(fmap1=fmap1, fmap2=fmap2, net0=net.permute(0, 2, 3, 1), inp=inp.permute(0, 2, 3, 1),
                 corr=[], net=[], mask=[], delta=[], coords=[]) if return_intermediates else None
    preds = []
    for _ in range(iters):                                                  # :93
        corr = corr_block.retrieve(coords1)                                 # :95
        flow = coords1 - coords0                                            # :97
        if variant == 'raft':
            net, mask, delta = basic_update_block(ops, net, inp, corr.permute(0, 3, 1, 2), flow.permute(0, 3, 1, 2))
        else:
            net, mask, delta = small_update_block(ops, net, inp, corr.permute(0, 3, 1, 2), flow.permute(0, 3, 1, 2))
        coords1 = coords1 + delta.permute(0, 2, 3, 1)                       # :102
        if variant == 'raft':
            up = upsample_flow(coords1 - coords0, mask.permute(0, 2, 3, 1))  # :105
        else:
            up = upflow8(coords1 - coords0)                                 # :223
        preds.append(up)
        if inter is not None:
            inter['corr'].append(corr)
            inter['net'].append(net.permute(0, 2, 3, 1))
            inter['mask'].append(None if mask is None else mask.permute(0, 2, 3, 1))
            inter['delta'].append(delta.permute(0, 2, 3, 1))
            inter['coords'].append(coords1)
    if return_intermediates:
        inter['corr_pyramid'] = corr_block.corr_pyramid
        return preds, inter
    return preds


def tf32_trunc(x):
    """Emulate a tensor core reading fp32 as TF32 (low 13 mantissa bits dropped)."""
    if x.dtype != torch.float32:
        return x
    return (x.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def tf32_round(x):
    """Round-to-nearest TF32 emulation."""
    if x.dtype != torch.float32:
        return x
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def bf16_round(x):
    return x.to(torch.bfloat16).to(x.dtype)
