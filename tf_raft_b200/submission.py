"""Benchmark submissions in RAFT's formats (RAFT evaluate.py create_sintel_submission / create_kitti_submission).

Both writers pad with RAFT's InputPadder (edge replication to a multiple of 8: centred for Sintel, at the bottom for
KITTI), predict, crop the flow back to the original frame and write one file per pair.  Frames are decoded on the
loader's threads and padded on the GPU (`FlowDataset.sequences` / `FlowDataset.batches`); the files are written on the
host.
"""
import os

import numpy as np
import torch

from .datasets import KITTI, MpiSintel
from .datasets.frame_utils import write_flow, write_flow_kitti
from .preprocess import placement

# write_flow_kitti stores uint16(64 * flow + 2^15): the flows whose code lies in [0, 65535], both ends exact in float32.
KITTI_FLOW_MIN = -512.0
KITTI_FLOW_MAX = (65535 - 2 ** 15) / 64.0


def _crop(pred, size, mode):
    H, W = pred.shape[-3:-1]
    top, left = placement(*size, H, W, mode)
    return pred[..., top:top + size[0], left:left + size[1], :]


def create_sintel_submission(model, root, output_path, *, dstypes=('clean', 'final'), warm_start=True, workers=4):
    """Flow for every pair of MPI Sintel's test split, written as `output_path/<dstype>/<scene>/frame%04d.flo`, the
    number being the pair's first frame index + 1, as RAFT names them.

    Each scene runs through `model.predict_video` at batch 1 on frames replicate-padded in Sintel mode.
    `warm_start=True` (RAFT's setting for its Sintel results) starts each pair after a scene's first from the
    forward-interpolated low-resolution flow of the previous pair; the warm start resets at every scene.
    `warm_start=False` predicts every pair from zero flow.  -> the number of files written."""
    written = 0
    for dstype in dstypes:
        ds = MpiSintel(split='test', root=root, dstype=dstype)
        for frames, _, _, size, indices in ds.sequences(padding='replicate', pad_mode='sintel', workers=workers,
                                                        device=model.device):
            preds = model.predict_video((f[None] for f in frames), warm_start=warm_start)
            for index, pred in zip(indices, preds):
                scene, frame = ds.extra_info[index]
                out_dir = os.path.join(output_path, dstype, scene)
                os.makedirs(out_dir, exist_ok=True)
                write_flow(os.path.join(out_dir, 'frame%04d.flo' % (frame + 1)), _crop(pred[0], size, 'sintel').cpu().numpy())
                written += 1
    return written


def kitti_flow_for_png(flow):
    """The flow `write_flow_kitti` can store: NaN set to 0, then clamped to [-512, 511.984375], where
    64 * flow + 2^15 lies in [0, 65535].  RAFT's writer casts that value to uint16 unchecked, which NumPy leaves
    undefined outside the range."""
    return torch.clamp(torch.nan_to_num(flow, nan=0.0), KITTI_FLOW_MIN, KITTI_FLOW_MAX)


def create_kitti_submission(model, root, output_path, *, batch_size=1, workers=4):
    """Flow for every pair of KITTI 2015's testing split, written as `output_path/<frame_id>` (the first frame's file
    name) with `write_flow_kitti`.  Frames are replicate-padded in KITTI mode (all vertical padding at the bottom), and
    the flow is cropped back and clamped first (`kitti_flow_for_png`).  -> the number of files written."""
    ds = KITTI(split='testing', root=root)
    os.makedirs(output_path, exist_ok=True)
    index = 0
    for image1, image2, _, _, sizes in ds.batches(batch_size, padding='replicate', pad_mode='kitti', workers=workers,
                                                  device=model.device):
        pred = model([image1, image2], training=False, last_only=True)[-1]
        for k, size in enumerate(sizes):
            flow = kitti_flow_for_png(_crop(pred[k], size, 'kitti')).cpu().numpy()
            write_flow_kitti(os.path.join(output_path, ds.extra_info[index][0]), flow.astype(np.float32))
            index += 1
    return index
