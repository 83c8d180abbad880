"""Centred crop-or-pad to a multiple-of-8 frame size -- the only preprocessing the hot path depends on.

The model needs H and W divisible by 8 (SURVEY.md section 8, trap 7: `initialize_flow` uses `h // 8` while the
SAME-padded stride-2 encoder yields `ceil(h / 8)`), so the reference pads Sintel's 436x1024 frames to 448x1024 with
`tf.image.resize_with_crop_or_pad` before the forward and crops the predicted flow back
(tf_raft/datasets/dataset.py:323-334, tf_raft/training.py:73-81).  These helpers restate that op for torch tensors
(any device; pure indexing, no arithmetic), so BASELINE config 3 runs through the same API.

`InputPadder` is RAFT's evaluation padding instead: the smallest multiple of 8, filled by edge replication, which is
what published RAFT numbers use.  It and the evaluation loader pad on the GPU with raft_b200_pad_batch (csrc/pad.cuh),
one launch for every plane of a batch.
"""
import ctypes

import torch

from . import _lib

PAD_MODES = ('sintel', 'kitti')
ZERO, REPLICATE = 0, 1                 # raft_pad_mode
_DTYPES = {torch.uint8: 0, torch.float32: 1}


class _PadPlane(ctypes.Structure):
    """struct raft_pad_plane (include/raft_b200.h)."""
    _fields_ = [('src', ctypes.c_void_p), ('dst', ctypes.c_void_p), ('h', ctypes.c_int), ('w', ctypes.c_int),
                ('c', ctypes.c_int), ('H', ctypes.c_int), ('W', ctypes.c_int), ('top', ctypes.c_int),
                ('left', ctypes.c_int), ('dtype', ctypes.c_int), ('mode', ctypes.c_int)]


def pad_planes(jobs):
    """One raft_b200_pad_batch launch on the current stream.  jobs: [(src, dst, top, left, mode), ...] with src
    (h, w[, c]) and dst (H, W[, c]) contiguous CUDA tensors of one dtype (uint8 or float32) on one device; src pixel
    (0, 0) lands at (top, left) of dst (negative crops); mode ZERO or REPLICATE."""
    if not jobs:
        return
    arr = (_PadPlane * len(jobs))()
    device = jobs[0][1].device
    for p, (src, dst, top, left, mode) in zip(arr, jobs):
        for t in (src, dst):
            if not t.is_cuda:
                raise RuntimeError('tf_raft_b200 pads CUDA tensors only (sm_90a); got a CPU tensor. '
                                   'There is no CPU fallback for this path.')
            if t.device != device:
                raise ValueError(f'pad_planes: tensors on {t.device} and {device}')
            if not t.is_contiguous():
                raise ValueError('pad_planes: expected contiguous tensors')
        if src.dtype != dst.dtype or src.dtype not in _DTYPES:
            raise TypeError(f'pad_planes: expected uint8 or float32 source and destination of one dtype, got '
                            f'{src.dtype} and {dst.dtype}')
        c = src.shape[2] if src.dim() == 3 else 1
        if src.dim() not in (2, 3) or dst.dim() != src.dim() or (dst.shape[2] if dst.dim() == 3 else 1) != c:
            raise ValueError(f'pad_planes: expected (h, w[, c]) planes of one channel count, got {tuple(src.shape)} '
                             f'and {tuple(dst.shape)}')
        p.src, p.dst = src.data_ptr(), dst.data_ptr()
        p.h, p.w, p.c, p.H, p.W = src.shape[0], src.shape[1], c, dst.shape[0], dst.shape[1]
        p.top, p.left, p.dtype, p.mode = int(top), int(left), _DTYPES[src.dtype], int(mode)
    arr_dev = torch.frombuffer(bytearray(arr), dtype=torch.uint8).pin_memory().to(device, non_blocking=True)
    _lib.call('pad_batch', device, arr, _lib.ptr(arr_dev), len(jobs))


def input_padding(h, w, mode='sintel'):
    """RAFT's InputPadder offsets of an h x w frame -> (top, bottom, left, right): the padding to the smallest multiple
    of 8 at or above each size, split evenly (the odd pixel after) -- except that mode 'kitti' puts all vertical
    padding at the bottom."""
    if mode not in PAD_MODES:
        raise ValueError(f'unknown pad mode {mode!r}; expected one of {PAD_MODES}')
    ph = (((h // 8) + 1) * 8 - h) % 8
    pw = (((w // 8) + 1) * 8 - w) % 8
    top = 0 if mode == 'kitti' else ph // 2
    return top, ph - top, pw // 2, pw - pw // 2


def placement(h, w, target_height, target_width, mode='sintel'):
    """(top, left) of an h x w source inside a target_height x target_width frame (negative = crop): centred as
    `resize_with_crop_or_pad` places it, except that mode 'kitti' pads at the bottom only."""
    if mode not in PAD_MODES:
        raise ValueError(f'unknown pad mode {mode!r}; expected one of {PAD_MODES}')
    ch, ph = _offsets(h, target_height)
    cw, pw = _offsets(w, target_width)
    top = -ch if ch else (0 if mode == 'kitti' else ph)
    return top, -cw if cw else pw


class InputPadder:
    """RAFT's InputPadder for (B, H, W, C) tensors (RAFT core/utils/utils.py): pads H and W to the smallest multiple of
    8 by edge replication (`F.pad(..., mode='replicate')`), centred in mode 'sintel', all vertical padding at the bottom
    in mode 'kitti' (see `input_padding`).  `shape` is the shape of the tensors to pad, (..., H, W, C)."""

    def __init__(self, shape, mode='sintel'):
        if len(shape) < 3:
            raise ValueError(f'InputPadder: expected a (..., H, W, C) shape, got {tuple(shape)}')
        self.ht, self.wd = int(shape[-3]), int(shape[-2])
        self.mode = mode
        self._pad = input_padding(self.ht, self.wd, mode)

    @property
    def padded_size(self):
        top, bottom, left, right = self._pad
        return self.ht + top + bottom, self.wd + left + right

    def pad(self, *tensors):
        """-> a list of new (B, H', W', C) tensors, all of them padded by one kernel launch.  Each input is a (B, H, W,
        C) uint8 or float32 CUDA tensor of the size this padder was made for.  When H and W are already multiples of 8
        the inputs come back as they are."""
        for t in tensors:
            if not isinstance(t, torch.Tensor) or not t.is_cuda:
                raise RuntimeError('InputPadder pads CUDA tensors only (sm_90a); got a CPU tensor or a non-tensor. '
                                   'There is no CPU fallback for this path.')
            if t.dim() != 4 or tuple(t.shape[1:3]) != (self.ht, self.wd):
                raise ValueError(f'InputPadder: expected (B, {self.ht}, {self.wd}, C), got {tuple(t.shape)}')
            if t.dtype not in _DTYPES:
                raise TypeError(f'InputPadder: expected uint8 or float32, got {t.dtype}')
        if not any(self._pad):
            return list(tensors)
        H, W = self.padded_size
        top, _, left, _ = self._pad
        outs, jobs = [], []
        for t in tensors:
            t = t.contiguous()
            out = torch.empty((t.shape[0], H, W, t.shape[3]), dtype=t.dtype, device=t.device)
            jobs += [(t[b], out[b], top, left, REPLICATE) for b in range(t.shape[0])]
            outs.append(out)
        pad_planes(jobs)
        return outs

    def unpad(self, x):
        """The original H x W rectangle of a padded (..., H', W', C) tensor (a view)."""
        top, _, left, _ = self._pad
        return x[..., top:top + self.ht, left:left + self.wd, :]


def _offsets(size, target):
    """(crop offset, pad offset) of tf.image.resize_with_crop_or_pad along one axis: `max(-diff // 2, 0)` and
    `max(diff // 2, 0)` with Python floor division, diff = target - size."""
    diff = target - size
    return max(-diff // 2, 0), max(diff // 2, 0)


def resize_with_crop_or_pad(x, target_height, target_width):
    """`tf.image.resize_with_crop_or_pad(x, target_height, target_width)` for `(..., H, W, C)` tensors.

    Central crop where the input is larger, central zero padding where it is smaller (the odd pixel of an odd
    difference goes after / is cropped after, as in TF)."""
    if x.dim() < 3:
        raise ValueError('expected a (..., H, W, C) tensor')
    if target_height <= 0 or target_width <= 0:
        raise ValueError('target_height and target_width must be positive')
    h, w = x.shape[-3], x.shape[-2]
    ch, ph = _offsets(h, target_height)
    cw, pw = _offsets(w, target_width)
    keep_h, keep_w = min(h, target_height), min(w, target_width)
    cropped = x[..., ch:ch + keep_h, cw:cw + keep_w, :]
    if keep_h == target_height and keep_w == target_width:
        return cropped.contiguous()
    out = torch.zeros(x.shape[:-3] + (target_height, target_width, x.shape[-1]), dtype=x.dtype, device=x.device)
    out[..., ph:ph + keep_h, pw:pw + keep_w, :] = cropped
    return out


def CropOrPadder(target_size):
    """Reference datasets/dataset.py:323-334: returns `f(image1, image2, flow, valid)` that crop-or-pads all four
    (valid is `(..., H, W)` and is padded with zeros, i.e. padded pixels are invalid)."""
    th, tw = target_size

    def f(image1, image2, flow, valid):
        image1 = resize_with_crop_or_pad(image1, th, tw)
        image2 = resize_with_crop_or_pad(image2, th, tw)
        flow = resize_with_crop_or_pad(flow, th, tw)
        valid = resize_with_crop_or_pad(valid.unsqueeze(-1), th, tw).squeeze(-1)
        return image1, image2, flow, valid
    return f


def pad_to_multiple(x, multiple=8):
    """Smallest centred zero padding of `(..., H, W, C)` that makes H and W multiples of `multiple`; returns the
    padded tensor and the original `(H, W)` for `resize_with_crop_or_pad(flow, H, W)` afterwards."""
    h, w = x.shape[-3], x.shape[-2]
    th, tw = -(-h // multiple) * multiple, -(-w // multiple) * multiple
    return resize_with_crop_or_pad(x, th, tw), (h, w)
