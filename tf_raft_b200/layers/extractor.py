"""Feature / context encoders -- host-side mirror of tf_raft/layers/extractor.py (SURVEY.md 8(f) rank 1).

backend='native' (default): one call into libraft_b200.so (raft_b200_encoder_forward): every convolution on
the wgmma kernel, stride-2 convolutions via TMA elementStrides, norms as fused epilogues (BatchNorm in
inference) or deterministic reduction kernels (InstanceNorm).
backend='torch': IEEE-fp32 cuDNN convolutions through PyTorch with the reference's TensorFlow semantics
restated (Keras 'same' padding incl. the asymmetric stride-2 case, eps = 1e-3 norms) -- kept as an
independent GPU cross-check of the native path, never selected implicitly.
Parameter names are the reference's Keras attribute paths, kernels HWIO, NHWC tensors at the interface.
"""
import ctypes
import math
import os

import torch
import torch.nn.functional as F

from .. import _lib


def force_ieee_fp32():
    """fp32 convolutions must really be fp32: PyTorch's cuDNN default is TF32 (10-bit mantissa), which alone
    moves the final flow by ~1 px (DESIGN.md "Precision").  Process-wide torch setting."""
    try:
        torch.backends.cudnn.conv.fp32_precision = 'ieee'
        torch.backends.cuda.matmul.fp32_precision = 'ieee'
    except Exception:                      # older PyTorch: legacy switches
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False


force_ieee_fp32()


def _same_pads(n_in, k, s):
    n_out = -(-n_in // s)
    total = max((n_out - 1) * s + k - n_in, 0)
    return total // 2, total - total // 2


def _glorot(shape, gen):
    kh, kw, cin, cout = shape
    limit = math.sqrt(6.0 / (kh * kw * cin + kh * kw * cout))
    return torch.empty(shape).uniform_(-limit, limit, generator=gen)


class _Params:
    """Named parameter store shared by the layer classes below."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.params = {}
        self._nchw_cache = {}

    def add_conv(self, name, kh, kw, cin, cout, gen):
        self.params[name + '.kernel'] = _glorot((kh, kw, cin, cout), gen).to(self.device)
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
        for name in self.params:
            src = torch.as_tensor(params[prefix + name], dtype=torch.float32)
            if tuple(src.shape) != tuple(self.params[name].shape):
                raise ValueError(f'{prefix + name}: expected {tuple(self.params[name].shape)}, got {tuple(src.shape)}')
            self.params[name] = src.to(self.device).contiguous()
        self._nchw_cache.clear()

    def conv(self, x, name, stride=1, padding='same'):
        """Keras Conv2D on an NCHW tensor (HWIO kernel, cross-correlation, TF padding rules)."""
        w = self._nchw_cache.get(name)
        if w is None:
            w = self.params[name + '.kernel'].permute(3, 2, 0, 1).contiguous()
            self._nchw_cache[name] = w
        if padding == 'same':
            pt, pb = _same_pads(x.shape[2], w.shape[2], stride)
            pl, pr = _same_pads(x.shape[3], w.shape[3], stride)
            if pt or pb or pl or pr:
                x = F.pad(x, (pl, pr, pt, pb))
        return F.conv2d(x, w, self.params[name + '.bias'], stride=stride)

    def norm(self, x, name, norm_type, training):
        eps = 1e-3        # tfa InstanceNormalization and keras BatchNormalization both default to 1e-3
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


def Normalization(norm_type, groups=None):
    """Reference extractor.py:6-16: validates the norm type (group norm is never instantiated by the
    reference models and is not provided here)."""
    if norm_type in ('batch', 'instance', None):
        return norm_type
    if norm_type == 'group':
        raise NotImplementedError('GroupNormalization is not used by RAFT / SmallRAFT')
    raise ValueError(f'Invalid norm_type specified: {norm_type}')


class _Encoder:
    """Common body of BasicEncoder / SmallEncoder (reference extractor.py:88-175)."""
    _c0 = 0
    _stages = ()
    _variant = None

    def __init__(self, output_dim=128, norm_type='batch', drop_rate=0.0, *, device='cuda', seed=None, backend=None):
        self.backend = backend or os.environ.get('RAFT_B200_ENCODER', 'native')
        if self.backend not in ('native', 'torch'):
            raise ValueError(f'unknown encoder backend {self.backend!r}')
        self._prepared = None
        self._ws = {}
        self.output_dim = output_dim
        self.norm_type = Normalization(norm_type)
        self.drop_rate = drop_rate
        gen = torch.Generator(device='cpu')
        gen.manual_seed(0 if seed is None else seed)
        self.store = _Params(device)
        s = self.store
        s.add_conv('conv1', 7, 7, 3, self._c0, gen)
        s.add_norm('norm1', norm_type, self._c0)
        cin = self._c0
        for li, (c, stride) in enumerate(self._stages, start=1):
            for bi, st in enumerate((stride, 1)):
                p = f'layer{li}.{bi}'
                s.add_conv(p + '.conv1', 3, 3, cin, c, gen)
                s.add_conv(p + '.conv2', 3, 3, c, c, gen)
                s.add_norm(p + '.norm1', norm_type, c)
                s.add_norm(p + '.norm2', norm_type, c)
                if st != 1:
                    s.add_conv(p + '.downsample.0', 1, 1, cin, c, gen)
                    s.add_norm(p + '.downsample.1', norm_type, c)
                cin = c
        s.add_conv('conv2', 1, 1, cin, output_dim, gen)

    @property
    def params(self):
        return self.store.params

    def load_params(self, params, prefix=''):
        self.store.load(params, prefix)
        self._prepared = None

    def state_dict(self, prefix=''):
        return {prefix + k: v for k, v in self.store.params.items()}

    # -- native path --------------------------------------------------------------------------------
    def _conv_struct(self, name):
        k = self.store.params[name + '.kernel']
        return _lib.RaftConv(k.data_ptr(), self.store.params[name + '.bias'].data_ptr(), *k.shape)

    def _norm_struct(self, name):
        p = self.store.params
        if self.norm_type is None:
            return _lib.RaftNorm(None, None, None, None)
        mm = p.get(name + '.moving_mean')
        mv = p.get(name + '.moving_variance')
        return _lib.RaftNorm(p[name + '.gamma'].data_ptr(), p[name + '.beta'].data_ptr(),
                             None if mm is None else mm.data_ptr(), None if mv is None else mv.data_ptr())

    def prepared(self):
        if self._prepared is None:
            L = _lib.lib()
            w = _lib.RaftEncoderWeights()
            w.conv1 = self._conv_struct('conv1')
            w.norm1 = self._norm_struct('norm1')
            k = 0
            for li, (_, stride) in enumerate(self._stages, start=1):
                for bi, st in enumerate((stride, 1)):
                    p = f'layer{li}.{bi}'
                    blk = w.block[k]
                    blk.conv1, blk.conv2 = self._conv_struct(p + '.conv1'), self._conv_struct(p + '.conv2')
                    blk.norm1, blk.norm2 = self._norm_struct(p + '.norm1'), self._norm_struct(p + '.norm2')
                    if st != 1:
                        blk.downsample = self._conv_struct(p + '.downsample.0')
                        blk.downsample_norm = self._norm_struct(p + '.downsample.1')
                    k += 1
            w.conv2 = self._conv_struct('conv2')
            nbytes = ctypes.c_size_t()
            _lib.check(L.raft_b200_encoder_prepared_bytes(self._variant, self.output_dim, ctypes.byref(nbytes)),
                       'encoder_prepared_bytes')
            blob = _lib.workspace(nbytes.value, self.store.device)
            with torch.cuda.device(self.store.device):
                _lib.check(L.raft_b200_encoder_prepare(self._variant, _lib.NORM_TYPES[self.norm_type], self.output_dim,
                                                       ctypes.cast(ctypes.pointer(w), ctypes.c_void_p), _lib.ptr(blob),
                                                       blob.numel(), _lib.stream()), 'encoder_prepare')
            self._prepared = blob
        return self._prepared

    def _native(self, x, training, raw_image):
        x = _lib.f32c(x)
        n, h, w, c = x.shape
        if c != 3:
            raise ValueError(f'encoder input must be (N, H, W, 3); got {tuple(x.shape)}')
        L = _lib.lib()
        key = (n, h, w)
        if key not in self._ws:
            nbytes = ctypes.c_size_t()
            _lib.check(L.raft_b200_encoder_workspace_bytes(self._variant, n, h, w, ctypes.byref(nbytes)),
                       'encoder_workspace_bytes')
            self._ws = {key: _lib.workspace(nbytes.value, x.device)}
        ws = self._ws[key]
        out = torch.empty((n, -(-h // 8), -(-w // 8), self.output_dim), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(L.raft_b200_encoder_forward(self._variant, _lib.NORM_TYPES[self.norm_type], self.output_dim,
                                                   _lib.ptr(self.prepared()), _lib.ptr(x), n, h, w, int(bool(training)),
                                                   int(bool(raw_image)), _lib.ptr(out), _lib.ptr(ws), ws.numel(),
                                                   _lib.stream()), 'encoder_forward')
        return out

    def _res_block(self, x, p, stride, training):
        """Reference ResBlock.call, extractor.py:41-49."""
        s, nt = self.store, self.norm_type
        fx = F.relu(s.norm(s.conv(x, p + '.conv1', stride), p + '.norm1', nt, training))
        fx = F.relu(s.norm(s.conv(fx, p + '.conv2', 1), p + '.norm2', nt, training))
        if stride != 1:
            x = s.norm(s.conv(x, p + '.downsample.0', stride, padding='valid'), p + '.downsample.1', nt, training)
        return F.relu(x + fx)

    def __call__(self, inputs, training=False, *, raw_image=False):
        """NHWC tensor, or a list/tuple of two (concatenated along the batch, split on return).

        `raw_image=True` (keyword-only extra): inputs are 0..255 images and the 2*(x/255)-1 of model.py:70-71
        is applied inside (fused into the first load on the native path)."""
        is_list = isinstance(inputs, (tuple, list))
        x = torch.cat(list(inputs), dim=0) if is_list else inputs
        if self.backend == 'native' and not (self.drop_rate > 0 and training):
            out = self._native(x, training, raw_image)
            if is_list:
                n = out.shape[0] // 2
                return [out[:n], out[n:]]
            return out
        if raw_image:
            x = 2 * (x / 255.0) - 1.0
        x = x.permute(0, 3, 1, 2)
        s, nt = self.store, self.norm_type
        x = F.relu(s.norm(s.conv(x, 'conv1', 2), 'norm1', nt, training))
        for li, (_, stride) in enumerate(self._stages, start=1):
            x = self._res_block(x, f'layer{li}.0', stride, training)
            x = self._res_block(x, f'layer{li}.1', 1, training)
        x = s.conv(x, 'conv2', 1, padding='valid')
        if self.drop_rate > 0 and training:
            x = F.dropout(x, self.drop_rate, training=True)
        x = x.permute(0, 2, 3, 1).contiguous()
        if is_list:
            n = x.shape[0] // 2
            return [x[:n].contiguous(), x[n:].contiguous()]
        return x


class BasicEncoder(_Encoder):
    """Reference extractor.py:88-130."""
    _c0 = 64
    _stages = ((64, 1), (96, 2), (128, 2))
    _variant = _lib.VARIANT_BASIC


class SmallEncoder(_Encoder):
    """Reference extractor.py:133-175 (built from ResBlocks, not bottlenecks)."""
    _c0 = 32
    _stages = ((32, 1), (64, 2), (96, 2))
    _variant = _lib.VARIANT_SMALL
