"""Named parameter store of the encoders, the update blocks and the stand-alone update layers.

Parameter names are the reference's Keras attribute paths, kernels HWIO as Keras stores them.  The seeded default
values are drawn on the CPU in the order of the `add_conv` calls, so they depend on the seed and the layer alone.
`conventions` selects the torch backend's arithmetic: 'tf-raft' (Keras 'same' padding, eps 1e-3) or 'pytorch' (the
original RAFT's symmetric padding, eps 1e-5).
"""
import math

import torch
import torch.nn.functional as F


def _same_pads(n_in, k, s):
    n_out = -(-n_in // s)
    total = max((n_out - 1) * s + k - n_in, 0)
    return total // 2, total - total // 2


class _Params:
    def __init__(self, device, seed, conventions='tf-raft'):
        self.device = torch.device(device)
        self.conventions = conventions
        self.params = {}
        self._gen = torch.Generator(device='cpu')
        self._gen.manual_seed(0 if seed is None else seed)
        self._nchw_cache = {}

    def add_conv(self, name, kh, kw, cin, cout):
        """Keras defaults: glorot-uniform kernel U(-l, l), l = sqrt(6 / (fan_in + fan_out)), and zero bias."""
        limit = math.sqrt(6.0 / (kh * kw * cin + kh * kw * cout))
        kernel = torch.empty(kh, kw, cin, cout).uniform_(-limit, limit, generator=self._gen)
        self.params[name + '.kernel'] = kernel.to(self.device)
        self.params[name + '.bias'] = torch.zeros(cout, device=self.device)

    def add_norm(self, name, norm_type, c):
        if norm_type is None:
            return
        self.params[name + '.gamma'] = torch.ones(c, device=self.device)
        self.params[name + '.beta'] = torch.zeros(c, device=self.device)
        if norm_type == 'batch':
            self.params[name + '.moving_mean'] = torch.zeros(c, device=self.device)
            self.params[name + '.moving_variance'] = torch.ones(c, device=self.device)

    def load(self, params, prefix=''):
        """Copy `{prefix+name: array}` (NumPy or torch, HWIO kernels) into the store."""
        for name in self.params:
            src = torch.as_tensor(params[prefix + name], dtype=torch.float32)
            if tuple(src.shape) != tuple(self.params[name].shape):
                raise ValueError(f'{prefix + name}: expected {tuple(self.params[name].shape)}, got {tuple(src.shape)}')
            self.params[name] = src.to(self.device).contiguous()
        self._nchw_cache.clear()

    def state_dict(self, prefix=''):
        return {prefix + k: v for k, v in self.params.items()}

    # -- the encoders' torch backend ------------------------------------------------------------------
    def conv(self, x, name, stride=1, padding='same'):
        """Keras Conv2D on an NCHW tensor (HWIO kernel, cross-correlation, TF padding rules)."""
        w = self._nchw_cache.get(name)
        if w is None:
            w = self.params[name + '.kernel'].permute(3, 2, 0, 1).contiguous()
            self._nchw_cache[name] = w
        if padding == 'same' and self.conventions == 'pytorch':         # nn.Conv2d(padding=(k-1)//2)
            return F.conv2d(x, w, self.params[name + '.bias'], stride=stride,
                            padding=((w.shape[2] - 1) // 2, (w.shape[3] - 1) // 2))
        if padding == 'same':
            pt, pb = _same_pads(x.shape[2], w.shape[2], stride)
            pl, pr = _same_pads(x.shape[3], w.shape[3], stride)
            if pt or pb or pl or pr:
                x = F.pad(x, (pl, pr, pt, pb))
        return F.conv2d(x, w, self.params[name + '.bias'], stride=stride)

    def norm(self, x, name, norm_type, training):
        # tfa InstanceNormalization and keras BatchNormalization both default to 1e-3, nn.InstanceNorm2d / BatchNorm2d to 1e-5
        eps = 1e-5 if self.conventions == 'pytorch' else 1e-3
        if norm_type is None:
            return x
        g = self.params[name + '.gamma'].view(1, -1, 1, 1)
        b = self.params[name + '.beta'].view(1, -1, 1, 1)
        if norm_type == 'instance':
            mean = x.mean(dim=(2, 3), keepdim=True)
            var = x.var(dim=(2, 3), unbiased=False, keepdim=True)
        elif norm_type == 'batch':
            if training:
                mean = x.mean(dim=(0, 2, 3), keepdim=True)
                var = x.var(dim=(0, 2, 3), unbiased=False, keepdim=True)
                mom, n = 0.99, x.shape[0] * x.shape[2] * x.shape[3]      # keras fused update: n / (n - 1) (DESIGN.md §9)
                self.params[name + '.moving_mean'].mul_(mom).add_((1 - mom) * mean.flatten())
                self.params[name + '.moving_variance'].mul_(mom).add_((1 - mom) * n / max(n - 1, 1) * var.flatten())
            else:
                mean = self.params[name + '.moving_mean'].view(1, -1, 1, 1)
                var = self.params[name + '.moving_variance'].view(1, -1, 1, 1)
        else:
            raise ValueError(f'Invalid norm_type specified: {norm_type}')
        return (x - mean) * torch.rsqrt(var + eps) * g + b
