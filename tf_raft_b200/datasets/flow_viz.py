"""Flow colour-wheel visualisation on the GPU -- mirror of tf_raft/datasets/flow_viz.py (Baker et al., "A Database and
Evaluation Methodology for Optical Flow", ICCV 2007: the Middlebury colour coding).

`flow_to_image` and `flow_uv_to_colors` take CUDA tensors and return uint8 images on the same device; the colouring is
raft_b200_flow_to_image (csrc/flow_viz.cuh).  It follows the reference's NumPy 2 arithmetic step for step (DESIGN.md
section 3.5), with a correctly rounded atan2 where NumPy's float32 arctan2 depends on the build.  `make_colorwheel` is
the host-side table, as in the reference.
"""
import numpy as np
import torch

from .. import _lib

_FLOWVIZ_INF, _FLOWVIZ_NAN, _FLOWVIZ_BAD_RAD_MAX = 1, 2, 4
_FLT_MAX = float(np.finfo(np.float32).max)          # clip_flow and rad_max go to the kernels as float32
_SEGMENTS = ((15, 'RY'), (6, 'YG'), (4, 'GC'), (11, 'CB'), (13, 'BM'), (6, 'MR'))


def make_colorwheel():
    """flow_viz.py:20-67: the (55, 3) float64 colour wheel, ramps RY 15, YG 6, GC 4, CB 11, BM 13, MR 6, each step
    floor(255 * j / n)."""
    wheel = np.zeros((55, 3))
    col = 0
    for n, name in _SEGMENTS:
        ramp = np.floor(255 * np.arange(n) / n)
        rising, channel = {'RY': (True, 1), 'YG': (False, 0), 'GC': (True, 2), 'CB': (False, 1), 'BM': (True, 0),
                           'MR': (False, 2)}[name]
        full = {'RY': 0, 'YG': 1, 'GC': 1, 'CB': 2, 'BM': 2, 'MR': 0}[name]
        wheel[col:col + n, full] = 255
        wheel[col:col + n, channel] = ramp if rising else 255 - ramp
        col += n
    return wheel


def _planes(x, what):
    if not isinstance(x, torch.Tensor):
        raise TypeError(f'{what}: expected a torch tensor, got {type(x).__name__}')
    if not x.is_cuda:
        raise RuntimeError('tf_raft_b200 runs on CUDA tensors only (sm_90a); got a CPU tensor. '
                           'There is no CPU fallback for this path.')
    if not x.is_floating_point():
        raise ValueError(f'{what}: expected a floating-point tensor, got {x.dtype}')
    return x.to(torch.float32).contiguous()


def _run(u, v, stride, b, h, w, clip_flow, normalize, rad_max, bgr, device):
    if h * w == 0 or b == 0:
        raise ValueError(f'empty image ({b} x {h} x {w})')
    if b > 65535 or h * w >= 2 ** 31:
        raise ValueError(f'too large: {b} images of {h} x {w} pixels')
    image = torch.empty((b, h, w, 3), dtype=torch.uint8, device=device)
    status = torch.empty(b, dtype=torch.int32, device=device)
    work = torch.empty(b, dtype=torch.int32, device=device) if normalize and rad_max is None else None
    clip = clip_flow is not None
    _lib.call('flow_to_image', device, _lib.ptr(u), _lib.ptr(v), stride, b, h, w, int(clip),
              float(clip_flow) if clip else 0.0, int(normalize), _lib.ptr(rad_max), int(bool(bgr)), _lib.ptr(image),
              _lib.ptr(work), _lib.ptr(status))
    return image, status.cpu()                                   # the one synchronisation of a call


def flow_uv_to_colors(u, v, convert_to_bgr=False):
    """flow_viz.py:70-106: colours of (H, W) or (B, H, W) flow components u, v (CUDA tensors, taken as float32) ->
    uint8 (..., H, W, 3) on the same device, RGB or BGR.  |(u, v)| <= 1 fades towards white at the centre, larger
    magnitudes are darkened by 0.75.  NaN in u or v raises ValueError naming the image (the reference fails with
    IndexError); +-inf is coloured, as in the reference."""
    u, v = _planes(u, 'flow_uv_to_colors'), _planes(v, 'flow_uv_to_colors')
    if u.shape != v.shape or u.dim() not in (2, 3):
        raise ValueError(f'flow_uv_to_colors: expected u, v of one (H, W) or (B, H, W) shape, got {tuple(u.shape)} '
                         f'and {tuple(v.shape)}')
    if u.device != v.device:
        raise ValueError(f'flow_uv_to_colors: u is on {u.device}, v on {v.device}')
    single = u.dim() == 2
    b, h, w = (1,) + tuple(u.shape) if single else tuple(u.shape)
    image, status = _run(u, v, 1, b, h, w, None, False, None, convert_to_bgr, u.device)
    bad = torch.nonzero(status & _FLOWVIZ_NAN)
    if len(bad):
        raise ValueError(f'flow_uv_to_colors: image {int(bad[0])} has NaN flow components')
    return image[0] if single else image


def flow_to_image(flow_uv, clip_flow=None, convert_to_bgr=False, *, rad_max=None):
    """flow_viz.py:109-132: (H, W, 2) or (B, H, W, 2) flow (CUDA, taken as float32) -> uint8 (H, W, 3) or (B, H, W, 3)
    on the same device.  Each image is clipped to [0, clip_flow] when clip_flow is given, normalised by its own largest
    flow magnitude (plus 1e-5) and coloured by `flow_uv_to_colors`; out[b] equals the call on flow_uv[b] alone.

    rad_max (keyword-only, an addition beyond the reference): a float, or a (B,) tensor on the flow's device, that
    replaces each image's own maximum, so that the frames of a video share one scale instead of flickering.  Pixels
    beyond it come out darkened (the reference's 0.75 branch).  It must be finite and >= 0.

    Raises ValueError for a wrong shape, an empty image, a negative or non-finite clip_flow or rad_max, and for flow
    with a NaN or +-inf component after the clip, naming the first such image (where the reference fails with
    IndexError or on an empty max).  Checking reads the B status words back: one synchronisation per call."""
    flow = _planes(flow_uv, 'flow_to_image')
    if flow.dim() not in (3, 4) or flow.shape[-1] != 2:
        raise ValueError(f'flow_to_image: expected an (H, W, 2) or (B, H, W, 2) flow, got {tuple(flow.shape)}')
    single = flow.dim() == 3
    if single:
        flow = flow.unsqueeze(0)
    b, h, w, _ = flow.shape
    if clip_flow is not None:
        clip_flow = float(clip_flow)
        if not (0.0 <= clip_flow <= _FLT_MAX):
            raise ValueError(f'flow_to_image: clip_flow must be finite and >= 0, got {clip_flow}')
    if rad_max is not None:
        if isinstance(rad_max, torch.Tensor):
            if rad_max.device != flow.device or rad_max.shape not in ((b,), ()):
                raise ValueError(f'flow_to_image: rad_max must be a float or a ({b},) tensor on {flow.device}, got '
                                 f'{tuple(rad_max.shape)} on {rad_max.device}')
            rad_max = rad_max.to(torch.float32).expand(b).contiguous()
        else:
            r = float(rad_max)
            if not (0.0 <= r <= _FLT_MAX):
                raise ValueError(f'flow_to_image: rad_max must be finite and >= 0, got {rad_max}')
            rad_max = torch.full((b,), r, dtype=torch.float32, device=flow.device)
    u = flow.reshape(-1)                                         # u at even, v at odd floats: stride 2
    image, status = _run(u, u[1:], 2, b, h, w, clip_flow, True, rad_max, convert_to_bgr, flow.device)
    bad = torch.nonzero(status & _FLOWVIZ_BAD_RAD_MAX)
    if len(bad):
        raise ValueError(f'flow_to_image: rad_max of image {int(bad[0])} is negative or not finite')
    bad = torch.nonzero(status & (_FLOWVIZ_INF | _FLOWVIZ_NAN))
    if len(bad):
        raise ValueError(f'flow_to_image: image {int(bad[0])} has a NaN or infinite flow component'
                         + (' after clipping' if clip_flow is not None else ''))
    return image[0] if single else image
