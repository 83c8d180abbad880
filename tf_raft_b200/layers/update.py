"""Update blocks -- host-side mirror of tf_raft/layers/update.py.

`BasicUpdateBlock(filters=128)([net, inp, corr, flow]) -> (net, 0.25*mask, delta_flow)` and
`SmallUpdateBlock(filters=96)(...) -> (net, None, delta_flow)` keep the reference's list-of-4 in /
tuple-of-3 out contract (update.py:118-125, 143-153).  Inside the blocks the motion encoder, (Sep)ConvGRU,
flow head and mask head are one launch sequence in libraft_b200.so (raft_b200_update_basic /
raft_b200_update_small); `FlowHead`, `ConvGRU`, `SepConvGRU`, `SmallMotionEncoder`, `BasicMotionEncoder`
are also provided as stand-alone layers (bottom of this file) for code that builds them one by one.

Parameters live in `self.params`, keyed by the reference's Keras attribute paths relative to the
block ('encoder.convc1.kernel', 'gru.convz1.bias', 'flow_head.conv1.kernel', 'mask.0.kernel', ...),
kernels in HWIO layout exactly as Keras stores them.
"""
import ctypes

import torch

from .. import _lib
from ._params import _Params

# (name, kh, kw, cin, cout) in the member order of raft_basic_weights / raft_small_weights.
BASIC_CONVS = (
    ('encoder.convc1', 1, 1, 324, 256), ('encoder.convc2', 3, 3, 256, 192), ('encoder.convf1', 7, 7, 2, 128),
    ('encoder.convf2', 3, 3, 128, 64), ('encoder.conv', 3, 3, 256, 126),
    ('gru.convz1', 1, 5, 384, 128), ('gru.convr1', 1, 5, 384, 128), ('gru.convq1', 1, 5, 384, 128),
    ('gru.convz2', 5, 1, 384, 128), ('gru.convr2', 5, 1, 384, 128), ('gru.convq2', 5, 1, 384, 128),
    ('flow_head.conv1', 3, 3, 128, 256), ('flow_head.conv2', 3, 3, 256, 2),
    ('mask.0', 3, 3, 128, 256), ('mask.2', 1, 1, 256, 576),
)
SMALL_CONVS = (
    ('encoder.convc1', 1, 1, 196, 96), ('encoder.convf1', 7, 7, 2, 64), ('encoder.convf2', 3, 3, 64, 32),
    ('encoder.conv', 3, 3, 128, 80),
    ('gru.convz', 3, 3, 242, 96), ('gru.convr', 3, 3, 242, 96), ('gru.convq', 3, 3, 242, 96),
    ('flow_head.conv1', 3, 3, 96, 128), ('flow_head.conv2', 3, 3, 128, 2),
)


class _ConvParams:
    """The parameters of the convolutions `_convs`, (name, kh, kw, cin, cout) each, initialised in that order."""
    _convs = ()

    def __init__(self, *, device=None, seed=None):
        self.device = torch.device('cuda' if device is None else device)
        self.store = _Params(self.device, seed)
        for conv in self._convs:
            self.store.add_conv(*conv)

    @property
    def params(self):
        return self.store.params

    def load_params(self, params, prefix=''):
        """Copy `{prefix+name: array}` (NumPy or torch, HWIO kernels) into the layer."""
        self.store.load(params, prefix)


class _UpdateBlock(_ConvParams):
    _variant = None
    _hidden = 0
    _context = 0
    _corr_ch = 0

    def __init__(self, filters, *, precision=None, device=None, seed=None):
        if filters != self._hidden:
            raise ValueError(f'{type(self).__name__} kernels are built for filters={self._hidden} '
                             f'(the only value the reference models use); got {filters}')
        self.filters = filters
        self.precision = _lib.resolve_precision(precision)
        super().__init__(device=device, seed=seed)
        self._prepared = None
        self.workspaces = _lib.WorkspaceCache()

    # -- parameters -------------------------------------------------------------------------
    def load_params(self, params, prefix=''):
        super().load_params(params, prefix)
        self._prepared = None

    def state_dict(self, prefix=''):
        return self.store.state_dict(prefix)

    def _weights_struct(self):
        arr = (_lib.RaftConv * len(self._convs))()
        for i, (name, kh, kw, cin, cout) in enumerate(self._convs):
            arr[i] = _lib.RaftConv(self.params[name + '.kernel'].data_ptr(), self.params[name + '.bias'].data_ptr(),
                                   kh, kw, cin, cout)
        return arr

    def prepared(self):
        """Device blob of re-laid-out weights (built once per parameter set)."""
        if self._prepared is None:
            nbytes = _lib.query_bytes('update_prepared_bytes', self._variant, self._corr_ch, self.precision)
            blob = _lib.workspace(nbytes, self.device)
            arr = self._weights_struct()
            _lib.call('update_prepare', blob.device, self._variant, ctypes.cast(arr, ctypes.c_void_p), _lib.ptr(blob),
                      blob.numel(), self.precision)
            self._prepared = blob
        return self._prepared

    def workspace(self, b, h, w):
        return self.workspaces.get((b, h, w), self.device, lambda: _lib.query_bytes(
            'update_workspace_bytes', self._variant, b, h, w, self.precision))

    def _check_inputs(self, inputs):
        net, inp, corr, flow = inputs
        net, inp, corr, flow = _lib.f32c(net), _lib.f32c(inp), _lib.f32c(corr), _lib.f32c(flow)
        b, h, w, c = net.shape
        for t, ch, nm in ((net, self._hidden, 'net'), (inp, self._context, 'inp'), (corr, self._corr_ch, 'corr'),
                          (flow, 2, 'flow')):
            if tuple(t.shape) != (b, h, w, ch):
                raise ValueError(f'{nm}: expected shape {(b, h, w, ch)}, got {tuple(t.shape)}')
        return net, inp, corr, flow, b, h, w


class BasicUpdateBlock(_UpdateBlock):
    """Reference update.py:128-153."""
    _convs = BASIC_CONVS
    _variant = _lib.VARIANT_BASIC
    _hidden, _context, _corr_ch = 128, 128, 324

    def __init__(self, filters=128, **kwargs):
        super().__init__(filters, **kwargs)

    def __call__(self, inputs, compute_mask=True):
        net, inp, corr, flow, b, h, w = self._check_inputs(inputs)
        net_out = torch.empty_like(net)
        mask = torch.empty((b, h, w, 576), dtype=torch.float32, device=net.device) if compute_mask else None
        delta = torch.empty((b, h, w, 2), dtype=torch.float32, device=net.device)
        ws = self.workspace(b, h, w)
        _lib.call('update_basic', net.device, _lib.ptr(self.prepared()), _lib.ptr(net), _lib.ptr(inp), _lib.ptr(corr),
                  _lib.ptr(flow), _lib.ptr(net_out), _lib.ptr(mask), _lib.ptr(delta), b, h, w, _lib.ptr(ws), ws.numel(),
                  self.precision)
        return net_out, mask, delta


class SmallUpdateBlock(_UpdateBlock):
    """Reference update.py:109-125."""
    _convs = SMALL_CONVS
    _variant = _lib.VARIANT_SMALL
    _hidden, _context, _corr_ch = 96, 64, 196

    def __init__(self, filters=96, **kwargs):
        super().__init__(filters, **kwargs)

    def __call__(self, inputs):
        net, inp, corr, flow, b, h, w = self._check_inputs(inputs)
        net_out = torch.empty_like(net)
        delta = torch.empty((b, h, w, 2), dtype=torch.float32, device=net.device)
        ws = self.workspace(b, h, w)
        _lib.call('update_small', net.device, _lib.ptr(self.prepared()), _lib.ptr(net), _lib.ptr(inp), _lib.ptr(corr),
                  _lib.ptr(flow), _lib.ptr(net_out), _lib.ptr(delta), b, h, w, _lib.ptr(ws), ws.numel(), self.precision)
        return net_out, None, delta


# ----------------------------------------------------------------------------------------------------------
# Stand-alone layers of update.py.  Inside RAFT they are fused into the update-block launch sequence above; these
# classes exist so that code which instantiates the reference's layers one by one keeps working.  Each Conv2D is one
# raft_b200_conv2d call (fp32 FFMA kernel); gating is elementwise on the same stream.
# ----------------------------------------------------------------------------------------------------------
_ACT = {None: 0, 'relu': 1, 'sigmoid': 2, 'tanh': 3}


class _ConvLayers(_ConvParams):
    def _conv(self, x, name, act=None, out=None, out_c0=0):
        x = _lib.f32c(x)
        k, b = self.params[name + '.kernel'], self.params[name + '.bias']
        kh, kw, cin, cout = k.shape
        bsz, h, w, c = x.shape
        if c != cin:
            raise ValueError(f'{name}: expected {cin} input channels, got {c}')
        if out is None:
            out = torch.empty((bsz, h, w, cout), dtype=torch.float32, device=x.device)
        _lib.call('conv2d', x.device, _lib.ptr(x), _lib.ptr(k), _lib.ptr(b), bsz, h, w, cin, kh, kw, cout, _ACT[act],
                  _lib.ptr(out), out.shape[-1], out_c0)
        return out


class FlowHead(_ConvLayers):
    """Reference update.py:5-14: conv2(relu(conv1(x))), 3x3 convolutions, 2 output channels."""

    def __init__(self, filters=256, in_channels=128, **kw):
        self.filters = filters
        self._convs = (('conv1', 3, 3, in_channels, filters), ('conv2', 3, 3, filters, 2))
        super().__init__(**kw)

    def __call__(self, inputs):
        return self._conv(self._conv(inputs, 'conv1', 'relu'), 'conv2')


class ConvGRU(_ConvLayers):
    """Reference update.py:17-35: 3x3 ConvGRU on [h, x]."""
    _taps = (('', 3, 3),)

    def __init__(self, filters=128, in_channels=None, **kw):
        self.filters = filters
        cin = filters + (in_channels if in_channels is not None else {96: 146, 128: 256}.get(filters, filters))
        self._convs = tuple((f'conv{g}{sfx}', kh, kwd, cin, filters) for sfx, kh, kwd in self._taps for g in 'zrq')
        super().__init__(**kw)

    def _step(self, h, x, sfx):
        hx = torch.cat([h, x], dim=-1)
        z = self._conv(hx, 'convz' + sfx, 'sigmoid')
        r = self._conv(hx, 'convr' + sfx, 'sigmoid')
        q = self._conv(torch.cat([r * h, x], dim=-1), 'convq' + sfx, 'tanh')
        return (1 - z) * h + z * q

    def __call__(self, inputs):
        h, x = inputs
        h, x = _lib.f32c(h), _lib.f32c(x)
        for sfx, _, _ in self._taps:
            h = self._step(h, x, sfx)
        return h


class SepConvGRU(ConvGRU):
    """Reference update.py:38-67: horizontal (1x5) then vertical (5x1) gated update."""
    _taps = (('1', 1, 5), ('2', 5, 1))


class SmallMotionEncoder(_ConvLayers):
    """Reference update.py:70-85 -> concat([conv(...), flow]) with 82 channels."""
    _convs = (('convc1', 1, 1, 196, 96), ('convf1', 7, 7, 2, 64), ('convf2', 3, 3, 64, 32), ('conv', 3, 3, 128, 80))

    def __call__(self, inputs):
        flow, corr = inputs
        cor = self._conv(corr, 'convc1', 'relu')
        flo = self._conv(self._conv(flow, 'convf1', 'relu'), 'convf2', 'relu')
        out = self._conv(torch.cat([cor, flo], dim=-1), 'conv', 'relu')
        return torch.cat([out, _lib.f32c(flow)], dim=-1)


class BasicMotionEncoder(_ConvLayers):
    """Reference update.py:88-106 -> concat([conv(...), flow]) with 128 channels."""
    _convs = (('convc1', 1, 1, 324, 256), ('convc2', 3, 3, 256, 192), ('convf1', 7, 7, 2, 128),
             ('convf2', 3, 3, 128, 64), ('conv', 3, 3, 256, 126))

    def __call__(self, inputs):
        flow, corr = inputs
        cor = self._conv(self._conv(corr, 'convc1', 'relu'), 'convc2', 'relu')
        flo = self._conv(self._conv(flow, 'convf1', 'relu'), 'convf2', 'relu')
        out = self._conv(torch.cat([cor, flo], dim=-1), 'conv', 'relu')
        return torch.cat([out, _lib.f32c(flow)], dim=-1)
