"""KITTI / HD1K flow PNGs decoded on the GPU (raft_b200_png16_flow_decode, csrc/dataset.cuh).

The host does the part that is already native: `frame_utils.inflate_png16` parses the chunks and inflates the IDAT
stream with zlib, and checks the row length and filter bytes.  One launch then undoes the PNG filters of a whole batch
of files, of any sizes, and writes the float32 flow and valid maps that `read_flow_kitti` returns.
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from .frame_utils import inflate_png16


class _Png16Image(ctypes.Structure):
    """struct raft_png16_image (include/raft_b200.h)."""
    _fields_ = [('offset', ctypes.c_size_t), ('h', ctypes.c_int), ('w', ctypes.c_int), ('flow', ctypes.c_void_p),
                ('valid', ctypes.c_void_p)]


def pack_rows(inflated):
    """Offsets of the inflated scanlines of `inflated` [(rows, h, w), ...] laid end to end -> (offsets, total bytes)."""
    offsets, off = [], 0
    for rows, _, _ in inflated:
        offsets.append(off)
        off += len(rows)
    return offsets, off


def decode_png16(data, layout, names, *, status_host=None):
    """Undo the PNG filters of several inflated flow PNGs already on the device, in one launch.

    data: uint8 CUDA tensor holding the scanlines; layout: [(offset, h, w), ...] into it; names: the files, for errors.
    -> [(flow (h, w, 2) float32, valid (h, w) float32), ...] on data's device, on the current stream.

    The kernel's per-image status is read back once.  With `status_host` (a pinned int32 tensor of len(layout)) the read
    is asynchronous: the caller later passes it to `check_png16_status`.  Otherwise this call waits for it."""
    n = len(layout)
    if n == 0:
        return []
    dev = data.device
    npix = [h * w for _, h, w in layout]
    out = torch.empty(3 * sum(npix), dtype=torch.float32, device=dev)     # every flow (8-byte aligned), then every valid
    arr = (_Png16Image * n)()
    result, fo, vo = [], 0, 2 * sum(npix)
    for i, ((offset, h, w), p) in enumerate(zip(layout, npix)):
        flow, valid = out[fo:fo + 2 * p].view(h, w, 2), out[vo:vo + p].view(h, w)
        fo, vo = fo + 2 * p, vo + p
        arr[i].offset, arr[i].h, arr[i].w = int(offset), int(h), int(w)
        arr[i].flow, arr[i].valid = flow.data_ptr(), valid.data_ptr()
        result.append((flow, valid))
    status = torch.empty(n, dtype=torch.int32, device=dev)
    arr_dev = torch.frombuffer(bytearray(arr), dtype=torch.uint8).to(dev, non_blocking=False)
    _lib.call('png16_flow_decode', dev, _lib.ptr(data), data.numel(), arr, _lib.ptr(arr_dev), n, _lib.ptr(status))
    if status_host is None:
        check_png16_status(status.cpu(), names)
    else:
        status_host.copy_(status, non_blocking=True)
    return result


def check_png16_status(status, names):
    """Raise ValueError naming the first file whose rows the kernel rejected (status = 1 + the bad row)."""
    bad = np.flatnonzero(status.numpy())
    if bad.size:
        i = int(bad[0])
        raise ValueError(f'{names[i]}: unknown PNG filter type in row {int(status[i]) - 1}')


def read_flow_kitti_batch(paths, device='cuda'):
    """`read_flow_kitti` for several equal-sized files, decoded on the GPU.
    -> (flow (n, H, W, 2) float32, valid (n, H, W) float32) on `device`.  Raises ValueError naming the file for a
    malformed PNG and for a size that differs from the first file's (`decode_png16` takes mixed sizes)."""
    paths = list(paths)
    if not paths:
        raise ValueError('read_flow_kitti_batch: no files')
    inflated = [inflate_png16(p) for p in paths]
    h, w = inflated[0][1:]
    for p, (_, hi, wi) in zip(paths, inflated):
        if (hi, wi) != (h, w):
            raise ValueError(f'{p}: {hi}x{wi}, but {paths[0]} is {h}x{w}; read_flow_kitti_batch needs equal sizes')
    offsets, total = pack_rows(inflated)
    host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for off, (rows, _, _) in zip(offsets, inflated):
        hv[off:off + len(rows)] = np.frombuffer(rows, dtype=np.uint8)
    data = host.to(device, non_blocking=True)
    decoded = decode_png16(data, [(off, h, w) for off in offsets], paths)
    return torch.stack([f for f, _ in decoded]), torch.stack([v for _, v in decoded])
