"""Feature / context encoders -- host-side mirror of tf_raft/layers/extractor.py (SURVEY.md 8(f) rank 1).

backend='native' (default): one call into libraft_b200.so (raft_b200_encoder_forward): every convolution on
the wgmma kernel, stride-2 convolutions via TMA elementStrides, norms as fused epilogues (BatchNorm in
inference) or deterministic reduction kernels (InstanceNorm).
backend='torch': IEEE-fp32 cuDNN convolutions through PyTorch with the reference's TensorFlow semantics
restated (Keras 'same' padding incl. the asymmetric stride-2 case, eps = 1e-3 norms) -- kept as an
independent GPU cross-check of the native path, never selected implicitly.
Parameter names are the reference's Keras attribute paths, kernels HWIO, NHWC tensors at the interface.
`conventions='pytorch'` (keyword-only) computes what the original PyTorch RAFT's encoders compute on both backends:
symmetric padding at stride 2 and eps = 1e-5 (include/raft_b200.h, raft_conventions).
`SmallEncoder(..., conventions='pytorch', blocks='bottleneck')` is the original RAFT-small's encoder: the same stem and
conv2 around six bottleneck blocks (1x1 -> 3x3 at the block's stride -> 1x1, widths 8, 16, 24), parameters named by the
original module paths (`layer2.0.conv3`, `layer2.0.downsample.0`, norms `norm1..3`, `downsample.1`).
"""
import ctypes
import os

import torch
import torch.nn.functional as F

from .. import _lib
from ._params import _Params


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
    _blocks = ('residual',)

    def __init__(self, output_dim=128, norm_type='batch', drop_rate=0.0, *, device='cuda', seed=None, backend=None,
                 conventions='tf-raft', blocks='residual'):
        self.backend = backend or os.environ.get('RAFT_B200_ENCODER', 'native')
        if self.backend not in ('native', 'torch'):
            raise ValueError(f'unknown encoder backend {self.backend!r}')
        if conventions not in _lib.CONVENTIONS:
            raise ValueError(f'unknown conventions {conventions!r}; expected one of {", ".join(_lib.CONVENTIONS)}')
        if blocks not in self._blocks:
            raise ValueError(f'{type(self).__name__}: unknown blocks {blocks!r}; expected one of {", ".join(self._blocks)}')
        if blocks == 'bottleneck':
            if conventions != 'pytorch':
                raise ValueError("blocks='bottleneck' is the original PyTorch RAFT-small's encoder and needs "
                                 "conventions='pytorch'; tf-raft's SmallEncoder is built from residual blocks")
            if norm_type not in ('instance', None):
                raise ValueError(f"blocks='bottleneck' takes norm_type 'instance' or None (the original RAFT-small's); "
                                 f'got {norm_type!r}')
            self._variant = _lib.VARIANT_SMALL_PYTORCH
        self.blocks = blocks
        self.conventions = conventions
        self._prepared = None
        self.workspaces = _lib.WorkspaceCache()
        self.output_dim = output_dim
        self.norm_type = Normalization(norm_type)
        self.drop_rate = drop_rate
        self.store = _Params(device, seed, conventions)
        s = self.store
        s.add_conv('conv1', 7, 7, 3, self._c0)
        s.add_norm('norm1', norm_type, self._c0)
        cin = self._c0
        for li, (c, stride) in enumerate(self._stages, start=1):
            for bi, st in enumerate((stride, 1)):
                p = f'layer{li}.{bi}'
                if blocks == 'bottleneck':
                    s.add_conv(p + '.conv1', 1, 1, cin, c // 4)
                    s.add_conv(p + '.conv2', 3, 3, c // 4, c // 4)
                    s.add_conv(p + '.conv3', 1, 1, c // 4, c)
                    for n, width in (('norm1', c // 4), ('norm2', c // 4), ('norm3', c)):
                        s.add_norm(f'{p}.{n}', norm_type, width)
                    if st != 1:
                        s.add_conv(p + '.downsample.0', 1, 1, cin, c)
                        s.add_norm(p + '.downsample.1', norm_type, c)
                    cin = c
                    continue
                s.add_conv(p + '.conv1', 3, 3, cin, c)
                s.add_conv(p + '.conv2', 3, 3, c, c)
                s.add_norm(p + '.norm1', norm_type, c)
                s.add_norm(p + '.norm2', norm_type, c)
                if st != 1:
                    s.add_conv(p + '.downsample.0', 1, 1, cin, c)
                    s.add_norm(p + '.downsample.1', norm_type, c)
                cin = c
        s.add_conv('conv2', 1, 1, cin, output_dim)

    @property
    def params(self):
        return self.store.params

    def load_params(self, params, prefix=''):
        self.store.load(params, prefix)
        self._prepared = None

    def state_dict(self, prefix=''):
        return self.store.state_dict(prefix)

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

    def _prepared_bottleneck(self, blob):
        w = _lib.RaftBottleneckEncoderWeights()
        w.conv1 = self._conv_struct('conv1')
        w.norm1 = self._norm_struct('norm1')
        k = 0
        for li, (_, stride) in enumerate(self._stages, start=1):
            for bi, st in enumerate((stride, 1)):
                p = f'layer{li}.{bi}'
                blk = w.block[k]
                blk.conv1, blk.conv2, blk.conv3 = (self._conv_struct(f'{p}.conv{i}') for i in (1, 2, 3))
                blk.norm1, blk.norm2, blk.norm3 = (self._norm_struct(f'{p}.norm{i}') for i in (1, 2, 3))
                if st != 1:
                    blk.downsample = self._conv_struct(p + '.downsample.0')
                    blk.downsample_norm = self._norm_struct(p + '.downsample.1')
                k += 1
        w.conv2 = self._conv_struct('conv2')
        _lib.call('encoder_prepare_bottleneck', blob.device, _lib.NORM_TYPES[self.norm_type], self.output_dim,
                  ctypes.cast(ctypes.pointer(w), ctypes.c_void_p), _lib.ptr(blob), blob.numel())

    def prepared(self):
        if self._prepared is None and self.blocks == 'bottleneck':
            blob = _lib.workspace(_lib.query_bytes('encoder_prepared_bytes', self._variant, self.output_dim),
                                  self.store.device)
            self._prepared_bottleneck(blob)
            self._prepared = blob
        if self._prepared is None:
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
            blob = _lib.workspace(_lib.query_bytes('encoder_prepared_bytes', self._variant, self.output_dim),
                                  self.store.device)
            _lib.call('encoder_prepare_ex', blob.device, self._variant, _lib.NORM_TYPES[self.norm_type], self.output_dim,
                      ctypes.cast(ctypes.pointer(w), ctypes.c_void_p), _lib.CONVENTIONS[self.conventions], _lib.ptr(blob),
                      blob.numel())
            self._prepared = blob
        return self._prepared

    def _native(self, x, training, raw_image):
        x = _lib.f32c(x)
        n, h, w, c = x.shape
        if c != 3:
            raise ValueError(f'encoder input must be (N, H, W, 3); got {tuple(x.shape)}')
        ws = self.workspaces.get((n, h, w), x.device,
                          lambda: _lib.query_bytes('encoder_workspace_bytes', self._variant, n, h, w))
        out = torch.empty((n, -(-h // 8), -(-w // 8), self.output_dim), dtype=torch.float32, device=x.device)
        _lib.call('encoder_forward', x.device, self._variant, _lib.NORM_TYPES[self.norm_type], self.output_dim,
                  _lib.ptr(self.prepared()), _lib.ptr(x), n, h, w, int(bool(training)), int(bool(raw_image)),
                  _lib.ptr(out), _lib.ptr(ws), ws.numel())
        return out

    def _res_block(self, x, p, stride, training):
        """Reference ResBlock.call, extractor.py:41-49."""
        s, nt = self.store, self.norm_type
        fx = F.relu(s.norm(s.conv(x, p + '.conv1', stride), p + '.norm1', nt, training))
        fx = F.relu(s.norm(s.conv(fx, p + '.conv2', 1), p + '.norm2', nt, training))
        if stride != 1:
            x = s.norm(s.conv(x, p + '.downsample.0', stride, padding='valid'), p + '.downsample.1', nt, training)
        return F.relu(x + fx)

    def _bottleneck_block(self, x, p, stride, training):
        """The original RAFT's BottleneckBlock.forward (symmetric padding through the store's 'pytorch' conventions)."""
        s, nt = self.store, self.norm_type
        y = F.relu(s.norm(s.conv(x, p + '.conv1', 1), p + '.norm1', nt, training))
        y = F.relu(s.norm(s.conv(y, p + '.conv2', stride), p + '.norm2', nt, training))
        y = F.relu(s.norm(s.conv(y, p + '.conv3', 1), p + '.norm3', nt, training))
        if stride != 1:
            x = s.norm(s.conv(x, p + '.downsample.0', stride, padding='valid'), p + '.downsample.1', nt, training)
        return F.relu(x + y)

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
        block = self._bottleneck_block if self.blocks == 'bottleneck' else self._res_block
        for li, (_, stride) in enumerate(self._stages, start=1):
            x = block(x, f'layer{li}.0', stride, training)
            x = block(x, f'layer{li}.1', 1, training)
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
    """Reference extractor.py:133-175 (built from ResBlocks); with conventions='pytorch', blocks='bottleneck' the
    original PyTorch RAFT-small's encoder (bottleneck blocks, norm 'instance' or None)."""
    _c0 = 32
    _stages = ((32, 1), (64, 2), (96, 2))
    _variant = _lib.VARIANT_SMALL
    _blocks = ('residual', 'bottleneck')
