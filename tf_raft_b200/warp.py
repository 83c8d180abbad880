"""Flow warping and flow composition on the GPU (additions: tf-raft has neither).

`warp` pulls an image, a feature map or a label map through a flow (backward warping); `compose_flow` chains two flows,
the step `RAFT.track_video` repeats along a clip.  Both sample with `fb_occlusion`'s rule: landing p = (x, y) + f,
closed frame [0, W-1] x [0, H-1], bilinear weights from floor(p), every operation one fp32 rounding with no FMA
(raft_b200_warp, raft_b200_compose_flow; DESIGN.md section 3.9).
"""
import ctypes

import torch

from . import _lib
from .layers.corr import _flow_field


def _flow(flow, what, name='flow'):
    if not isinstance(flow, torch.Tensor) or not flow.is_floating_point():
        raise TypeError(f'{what}: {name} must be a floating-point torch tensor, got '
                        f'{getattr(flow, "dtype", type(flow).__name__)}')
    flow = _flow_field(flow, what)
    return flow if flow.data_ptr() % 8 == 0 else flow.clone()      # the kernels load float2


def _mask(occ, shape, device, what, name):
    """An optional (B, H, W) mask as contiguous uint8 (nonzero = no correspondence), or None."""
    if occ is None:
        return None
    if not isinstance(occ, torch.Tensor) or occ.dtype not in (torch.bool, torch.uint8):
        raise TypeError(f'{what}: {name} must be a torch.bool or torch.uint8 tensor, got '
                        f'{getattr(occ, "dtype", type(occ).__name__)}')
    if tuple(occ.shape) != tuple(shape):
        raise ValueError(f'{what}: {name} {tuple(occ.shape)} does not match the flow\'s (B, H, W) {tuple(shape)}')
    if occ.device != device:
        raise ValueError(f'{what}: {name} is on {occ.device}, the flow on {device}')
    return occ.contiguous().view(torch.uint8)


def warp(src, flow, mode='bilinear', fill=0):
    """Backward warping: out[b, y, x] = src[b] sampled at (x, y) + flow[b, y, x].

    src: (B, Hs, Ws, C) CUDA tensor, floating point (computed in float32) or torch.uint8 (mode='nearest' only, for
    label and mask maps: labels come through unchanged).  flow: (B, H, W, 2) on the same device, in pixels of src; it
    sets the output grid and is not rescaled when src has another size.  mode: 'bilinear' (fb_occlusion's bilinear
    rule) or 'nearest' (the texel at floor(p + 0.5), clamped to the last row and column).

    Returns (out, occ): out (B, H, W, C) of src's dtype (float32 for floating src), equal to `fill` where the landing
    is outside src's closed frame [0, Ws-1] x [0, Hs-1] or not finite, and occ, torch.bool (B, H, W), True exactly
    there.  C from 1 to 1024."""
    what = 'warp'
    if not isinstance(src, torch.Tensor) or not (src.is_floating_point() or src.dtype == torch.uint8):
        raise TypeError(f'{what}: src must be a floating-point or uint8 torch tensor, got '
                        f'{getattr(src, "dtype", type(src).__name__)}')
    if mode not in _lib.WARP_MODES:
        raise ValueError(f'{what}: mode must be one of {sorted(_lib.WARP_MODES)}, got {mode!r}')
    flow = _flow(flow, what)
    u8 = src.dtype == torch.uint8
    if not src.is_cuda:
        _lib.f32c(src)                                                   # raises: no CPU fallback
    src = src.contiguous() if u8 else _lib.f32c(src)
    if src.dim() != 4:
        raise ValueError(f'{what}: expected a (B, Hs, Ws, C) src, got {tuple(src.shape)}')
    b, h, w, _ = flow.shape
    bs, hs, ws, c = src.shape
    if bs != b:
        raise ValueError(f'{what}: src batch {bs} and flow batch {b} differ')
    if src.device != flow.device:
        raise ValueError(f'{what}: src is on {src.device}, flow on {flow.device}')
    if not 1 <= c <= 1024:
        raise ValueError(f'{what}: src must have 1 to 1024 channels, got {c}')
    if u8:
        if mode != 'nearest':
            raise ValueError(f'{what}: uint8 src needs mode=\'nearest\' (bilinear would blend labels)')
        if not (isinstance(fill, int) and 0 <= fill <= 255):
            raise ValueError(f'{what}: fill for a uint8 src must be an integer 0..255, got {fill!r}')
    fill32 = ctypes.c_float(fill).value
    out = torch.empty((b, h, w, c), dtype=src.dtype, device=src.device)
    occ = torch.empty((b, h, w), dtype=torch.bool, device=src.device)
    _lib.call('warp', src.device, _lib.ptr(src), _lib.WARP_U8 if u8 else _lib.WARP_F32, hs, ws, c, _lib.ptr(flow), b, h,
              w, _lib.WARP_MODES[mode], fill32, _lib.ptr(out), _lib.ptr(occ))
    return out, occ


def compose_flow(f1, f2, occ1=None, occ2=None):
    """Chain two flows on one (B, H, W) grid: with p = x + f1(x),

        flow(x) = f1(x) + bilinear(f2, p),
        occ(x)  = occ1(x) or p outside the closed frame or occ2(nearest(p)) or flow(x) not finite,

    and flow(x) = f1(x) unchanged where occ(x) is True, so a lost track keeps its last position rather than NaN.
    f1, f2: (B, H, W, 2) CUDA flows; occ1, occ2: optional (B, H, W) torch.bool or uint8 masks (True / nonzero = no
    correspondence).  -> (flow, occ), a new float32 (B, H, W, 2) flow and a torch.bool (B, H, W) mask.

    Frame 0 -> t: acc, lost = compose_flow(acc, F_{t-1->t}, lost, occ_fw).  Frame t -> 0: acc, lost =
    compose_flow(B_{t->t-1}, acc, occ_bw, lost)."""
    what = 'compose_flow'
    f1, f2 = _flow(f1, what, 'f1'), _flow(f2, what, 'f2')
    if f1.shape != f2.shape:
        raise ValueError(f'{what}: f1 {tuple(f1.shape)} and f2 {tuple(f2.shape)} differ')
    if f1.device != f2.device:
        raise ValueError(f'{what}: f1 is on {f1.device}, f2 on {f2.device}')
    b, h, w, _ = f1.shape
    occ1 = _mask(occ1, (b, h, w), f1.device, what, 'occ1')
    occ2 = _mask(occ2, (b, h, w), f1.device, what, 'occ2')
    out = torch.empty_like(f1)
    occ = torch.empty((b, h, w), dtype=torch.bool, device=f1.device)
    _lib.call('compose_flow', f1.device, _lib.ptr(f1), _lib.ptr(f2), _lib.ptr(occ1), _lib.ptr(occ2), b, h, w,
              _lib.ptr(out), _lib.ptr(occ))
    return out, occ
