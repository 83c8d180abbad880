"""Correlation volume, pyramid and lookup -- host-side mirror of tf_raft/layers/corr.py.

Same names, argument meaning and error behaviour as the reference module, with torch CUDA
tensors in place of TF tensors.  Every function hands device pointers to libraft_b200.so
(include/raft_b200.h); nothing here computes on the host.
"""
import ctypes

import torch
import torch.nn.functional as F

from .. import _lib


def tfa_sampler(image, coords, mask=False):
    """Reference corr.py:6-25: `tfa.image.resampler` = ordinary bilinear interpolation with zero
    outside.  Not on the model's path (the reference never calls it); kept as the API alias."""
    if mask:
        raise NotImplementedError("mask is not implemented for True")
    m, h, w, _ = image.shape
    gx = 2 * coords[..., 0] / max(w - 1, 1) - 1
    gy = 2 * coords[..., 1] / max(h - 1, 1) - 1
    grid = torch.stack([gx, gy], dim=-1)
    out = F.grid_sample(image.permute(0, 3, 1, 2), grid, mode='bilinear', padding_mode='zeros', align_corners=True)
    return out.permute(0, 2, 3, 1)


def bilinear_sampler(image, coords):
    """Reference corr.py:28-69.  image (M, H, W, 1), coords (M, P, Q, 2) xy -> (M, P, Q, 1).

    floor/ceil corners: a sample whose clamped x or y is an integer is exactly 0."""
    image = _lib.f32c(image)
    coords = _lib.f32c(coords)
    m, h, w, c = image.shape
    if c != 1:
        raise ValueError('bilinear_sampler expects a single-channel image (M, H, W, 1)')
    p = coords.shape[1] * coords.shape[2]
    out = torch.empty(coords.shape[:-1] + (1,), dtype=torch.float32, device=image.device)
    _lib.call('bilinear_sampler', image.device, _lib.ptr(image), _lib.ptr(coords), m, h, w, p, _lib.ptr(out))
    return out


def coords_grid(batch_size, height, width, device=None):
    """Reference corr.py:72-90 -> (B, H, W, 2) with [..., 0] = x, [..., 1] = y."""
    device = torch.device('cuda') if device is None else torch.device(device)
    out = torch.empty((batch_size, height, width, 2), dtype=torch.float32, device=device)
    _lib.call('coords_grid', out.device, batch_size, height, width, _lib.ptr(out))
    return out


def _flow_field(flow, what):
    flow = _lib.f32c(flow)
    if flow.dim() != 4 or flow.shape[-1] != 2:
        raise ValueError(f'{what}: expected a (B, h, w, 2) flow, got {tuple(flow.shape)}')
    return flow


def forward_interpolate(flow):
    """RAFT's warm start for the next pair of a video (an addition: tf-raft has none).  (B, h, w, 2) -> (B, h, w, 2).

    Per image, source pixel (x, y) lands at (x + fx, y + fy) (fp64) and counts only strictly inside the frame,
    0 < x1 < w and 0 < y1 < h (NaN / inf flow never does).  Target pixel (X, Y) takes the flow of the landed source
    nearest to it (squared fp64 distance), ties to the lowest source index: scipy's
    `griddata((x1, y1), f, (X, Y), method='nearest')` with a deterministic tie rule.  Where griddata raises (no source
    lands inside the frame) the image gets zero flow.  Brute force on the GPU: O((h*w)^2) per image."""
    flow = _flow_field(flow, 'forward_interpolate')
    b, h, w, _ = flow.shape
    out = torch.empty_like(flow)
    _lib.call('forward_interpolate', flow.device, _lib.ptr(flow), b, h, w, _lib.ptr(out))
    return out


def fb_occlusion(flow_fw, flow_bw, alpha1=0.01, alpha2=0.5):
    """Forward-backward occlusion masks of bidirectional flow (an addition: tf-raft has none).

    flow_fw, flow_bw: (B, H, W, 2) flows a->b and b->a of B image pairs on one CUDA device -> (occ_fw, occ_bw), torch.bool
    (B, H, W).  occ_fw is True where pixel (x, y) of image a has no consistent correspondence in image b: its landing
    p = (x, y) + f leaves the closed frame [0, W-1] x [0, H-1], or, with g the bilinear sample of flow_bw at p,
    |f + g|^2 > alpha1 * (|f|^2 + |g|^2) + alpha2 (Sundaram, Brox and Keutzer, ECCV 2010, as used by UnFlow; the
    defaults are theirs).  occ_bw likewise with the roles swapped.  NaN anywhere in that computation counts as
    occluded.  Every operation is one fp32 rounding with no FMA (raft_b200_fb_occlusion, DESIGN.md section 3.5)."""
    for f in (flow_fw, flow_bw):
        if not isinstance(f, torch.Tensor) or not f.is_floating_point():
            raise TypeError(f'fb_occlusion: flows must be floating-point torch tensors, got '
                            f'{getattr(f, "dtype", type(f).__name__)}')
    flow_fw = _flow_field(flow_fw, 'fb_occlusion')
    flow_bw = _flow_field(flow_bw, 'fb_occlusion')
    if flow_fw.shape != flow_bw.shape:
        raise ValueError(f'fb_occlusion: flow_fw {tuple(flow_fw.shape)} and flow_bw {tuple(flow_bw.shape)} differ')
    if flow_fw.device != flow_bw.device:
        raise ValueError(f'fb_occlusion: flow_fw is on {flow_fw.device}, flow_bw on {flow_bw.device}')
    a1, a2 = ctypes.c_float(alpha1).value, ctypes.c_float(alpha2).value          # the kernel's fp32 thresholds
    if not (0.0 <= a1 < float('inf') and 0.0 <= a2 < float('inf')):
        raise ValueError(f'fb_occlusion: alpha1 and alpha2 must be finite and >= 0 in fp32, got {alpha1}, {alpha2}')
    # the kernel loads float2: a view starting at an odd float is copied to an aligned buffer
    flow_fw, flow_bw = (f if f.data_ptr() % 8 == 0 else f.clone() for f in (flow_fw, flow_bw))
    b, h, w, _ = flow_fw.shape
    occ_fw = torch.empty((b, h, w), dtype=torch.bool, device=flow_fw.device)
    occ_bw = torch.empty_like(occ_fw)
    _lib.call('fb_occlusion', flow_fw.device, _lib.ptr(flow_fw), _lib.ptr(flow_bw), b, h, w, a1, a2, _lib.ptr(occ_fw),
              _lib.ptr(occ_bw))
    return occ_fw, occ_bw


def coords_init(flow_init):
    """coords_grid(B, h, w) + flow_init in fp32: the iteration loop's entry state for a warm start (B, h, w, 2)."""
    flow_init = _flow_field(flow_init, 'coords_init')
    b, h, w, _ = flow_init.shape
    out = torch.empty_like(flow_init)
    _lib.call('coords_init', flow_init.device, _lib.ptr(flow_init), b, h, w, _lib.ptr(out))
    return out


def upflow8(flow, mode='bilinear'):
    """Reference corr.py:93-96: 8 * tf.image.resize(flow, (8h, 8w), 'bilinear') (half-pixel centres)."""
    if mode != 'bilinear':
        raise NotImplementedError("only mode='bilinear' is implemented")
    flow = _lib.f32c(flow)
    b, h, w, _ = flow.shape
    out = torch.empty((b, 8 * h, 8 * w, 2), dtype=torch.float32, device=flow.device)
    _lib.call('upflow8', flow.device, _lib.ptr(flow), b, h, w, _lib.ptr(out))
    return out


class CorrBlock:
    """Reference corr.py:99-162.  Plain class; the constructor builds the whole pyramid.

    Attributes as in the reference: fmap1, fmap2, num_levels, radius, corr_pyramid (list of
    `num_levels` tensors (B*h*w, h>>l, w>>l, 1)).  `precision` ('f16x2' tensor-core path, or 'fp32'
    CUDA-core path) is a keyword-only extra.
    """

    def __init__(self, fmap1, fmap2, num_levels=4, radius=4, *, precision=None):
        self.fmap1 = fmap1
        self.fmap2 = fmap2
        self.num_levels = num_levels
        self.radius = radius
        self.precision = _lib.resolve_precision(precision)
        f1, f2 = _lib.f32c(fmap1), _lib.f32c(fmap2)
        if f1.shape != f2.shape or f1.dim() != 4:
            raise ValueError(f'fmap1/fmap2 must both be (B, h, w, C); got {tuple(f1.shape)} and {tuple(f2.shape)}')
        b, h, w, c = f1.shape
        sizes = (ctypes.c_size_t * num_levels)()
        _lib.check(_lib.lib().raft_b200_corr_pyramid_sizes(b, h, w, num_levels, sizes), 'corr_pyramid_sizes')
        self.corr_pyramid = [torch.empty((b * h * w, h >> l, w >> l, 1), dtype=torch.float32, device=f1.device)
                             for l in range(num_levels)]
        ws = _lib.workspace(_lib.query_bytes('corr_workspace_bytes', b, h, w, c, num_levels, self.precision), f1.device)
        _lib.call('corr_pyramid_build', f1.device, _lib.ptr(f1), _lib.ptr(f2), b, h, w, c, num_levels,
                  _lib.ptr_array(self.corr_pyramid), _lib.ptr(ws), ws.numel(), self.precision)
        self._ws = ws          # keep alive until the stream has consumed it
        self._shape = (b, h, w)

    def retrieve(self, coords):
        """coords (B, h, w, 2) xy -> (B, h, w, num_levels*(2r+1)^2)."""
        coords = _lib.f32c(coords)
        b, h, w, _ = coords.shape
        if (b, h, w) != self._shape:
            raise ValueError(f'coords shape {tuple(coords.shape)} does not match the correlation volume {self._shape}')
        nch = self.num_levels * (2 * self.radius + 1) ** 2
        out = torch.empty((b, h, w, nch), dtype=torch.float32, device=coords.device)
        _lib.call('corr_lookup', coords.device, _lib.ptr_array(self.corr_pyramid), _lib.ptr(coords), b, h, w,
                  self.num_levels, self.radius, _lib.ptr(out), nch)
        return out

    def correlation(self, fmap1, fmap2):
        """Reference corr.py:154-162 -> (B, h, w, 1, h, w) = fmap1 . fmap2^T / sqrt(C)."""
        block = CorrBlock(fmap1, fmap2, num_levels=1, radius=self.radius, precision=self.precision)
        b, h, w = block._shape
        return block.corr_pyramid[0].reshape(b, h, w, 1, h, w)
