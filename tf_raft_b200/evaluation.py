"""Optical-flow metrics on the device and `evaluate`: EPE, the 1 / 3 / 5 px rates and KITTI's Fl-all.

`flow_metrics` runs raft_b200_flow_metrics (csrc/dataset.cuh): per image, int64 counts (n, epe < 1, epe < 3, epe < 5,
outliers) and an fp64 sum of the EPE over the kept pixels, in a fixed reduction order.  `FlowMetrics` keeps those
records on the device and aggregates them three ways:

- 'keras': the mean over batches of each batch's pooled ratios -- the reference's `EndPointError` metric, `test_step`
  and `fit(validation_data=...)` (tf_raft/losses/losses.py:24-85, model.py:146-159).
- 'pixel': pooled over every pixel -- RAFT's Sintel EPE (evaluate.py validate_sintel, with max_flow=None).
- 'image': EPE is the mean over images of each image's mean EPE; the 1 / 3 / 5 px rates and Fl-all = 100 * outliers /
  pixels are pooled -- RAFT's KITTI numbers (evaluate.py validate_kitti).

An outlier is epe > 3 and epe / |gt| > 0.05 (RAFT's validate_kitti).  A ratio over no pixels is NaN, as the reference's
mean of an empty tensor.
"""
import ctypes
import math

import numpy as np
import torch

from . import _lib

PROTOCOLS = ('keras', 'pixel', 'image')
_KEYS = ('epe', 'u1', 'u3', 'u5', 'fl_all')


def flow_metrics(pred, gt, valid=None, max_flow=400):
    """Per-image records of B flow pairs on the GPU, asynchronous.  pred, gt (B, H, W, 2) float32 CUDA tensors; valid
    (B, H, W) (nonzero = valid) or None; max_flow None turns the |gt| < max_flow test off.
    -> counts (B, 5) int64 [n, <1, <3, <5, outlier] and sums (B,) float64, on the device."""
    pred, gt = _lib.f32c(pred), _lib.f32c(gt)
    if pred.dim() != 4 or pred.shape[-1] != 2 or gt.shape != pred.shape:
        raise ValueError(f'flow_metrics: expected pred and gt of one (B, H, W, 2) shape, got {tuple(pred.shape)} and '
                         f'{tuple(gt.shape)}')
    B, H, W, _ = pred.shape
    if valid is not None:
        valid = _lib.f32c(torch.as_tensor(valid, device=gt.device))
        if tuple(valid.shape) != (B, H, W):
            raise ValueError(f'flow_metrics: expected valid of shape {(B, H, W)}, got {tuple(valid.shape)}')
    lib = _lib.lib()
    nbytes = ctypes.c_size_t()
    _lib.check(lib.raft_b200_flow_metrics_workspace_bytes(B, H, W, ctypes.byref(nbytes)), 'flow_metrics_workspace_bytes')
    counts = torch.empty((B, 5), dtype=torch.int64, device=gt.device)
    sums = torch.empty(B, dtype=torch.float64, device=gt.device)
    with torch.cuda.device(gt.device):
        ws = _lib.workspace(nbytes.value, gt.device)
        _lib.check(lib.raft_b200_flow_metrics(_lib.ptr(pred), _lib.ptr(gt), _lib.ptr(valid), B, H, W,
                                              int(max_flow is not None), float(0 if max_flow is None else max_flow),
                                              _lib.ptr(ws), ws.numel(), _lib.ptr(counts), _lib.ptr(sums),
                                              _lib.stream()), 'flow_metrics')
    return counts, sums


def _ratio(a, b):
    return float(a) / float(b) if b else math.nan


def aggregate(counts, sums, batch_sizes, protocol):
    """The three aggregations of per-image records (NumPy counts (N, 5), sums (N,)); batch_sizes splits the N images
    into the batches they were scored in ('keras' only).  -> {'epe', 'u1', 'u3', 'u5', 'fl_all' (percent), 'pixels'}."""
    if protocol not in PROTOCOLS:
        raise ValueError(f'unknown protocol {protocol!r}; expected one of {PROTOCOLS}')
    counts = np.asarray(counts, dtype=np.int64).reshape(-1, 5)
    sums = np.asarray(sums, dtype=np.float64).reshape(-1)
    n = counts[:, 0]
    pixels = int(n.sum())

    def pooled(c, s):
        tot, num = c.sum(axis=0), int(c[:, 0].sum())
        return {'epe': _ratio(s.sum(), num), 'u1': _ratio(tot[1], num), 'u3': _ratio(tot[2], num),
                'u5': _ratio(tot[3], num), 'fl_all': 100.0 * _ratio(tot[4], num)}

    if protocol == 'pixel':
        out = pooled(counts, sums)
    elif protocol == 'image':
        out = pooled(counts, sums)
        with np.errstate(invalid='ignore', divide='ignore'):
            out['epe'] = float(np.mean(sums / n)) if len(n) else math.nan
    else:
        if sum(batch_sizes) != len(n):
            raise ValueError(f'batch sizes add up to {sum(batch_sizes)}, but there are {len(n)} records')
        per, start = [], 0
        for b in batch_sizes:
            per.append(pooled(counts[start:start + b], sums[start:start + b]))
            start += b
        out = {k: (float(np.mean([p[k] for p in per])) if per else math.nan) for k in _KEYS}
    out['pixels'] = pixels
    return out


class FlowMetrics:
    """Accumulates per-image metric records on the device; `result()` reads them back once.

    max_flow: ground-truth pixels with |gt| >= max_flow are left out (None: none are); protocol: 'keras', 'pixel' or
    'image' (see the module docstring)."""

    def __init__(self, max_flow=400, protocol='keras'):
        if protocol not in PROTOCOLS:
            raise ValueError(f'unknown protocol {protocol!r}; expected one of {PROTOCOLS}')
        self.max_flow = max_flow
        self.protocol = protocol
        self.reset_states()

    def reset_states(self):
        self._counts, self._sums, self.batch_sizes = [], [], []

    def update_state(self, flow_gt, flow_pred, valid=None):
        """One batch: flow_gt, flow_pred (B, H, W, 2) and valid (B, H, W) on the GPU.  No host synchronisation."""
        counts, sums = flow_metrics(flow_pred, flow_gt, valid, self.max_flow)
        self._counts.append(counts)
        self._sums.append(sums)
        self.batch_sizes.append(int(counts.shape[0]))

    def records(self):
        """-> (counts (N, 5) int64, sums (N,) float64) as NumPy, one read-back."""
        if not self._counts:
            return np.zeros((0, 5), np.int64), np.zeros(0, np.float64)
        return torch.cat(self._counts).cpu().numpy(), torch.cat(self._sums).cpu().numpy()

    def result(self, protocol=None):
        counts, sums = self.records()
        return aggregate(counts, sums, self.batch_sizes, protocol or self.protocol)


def evaluate(model, dataset, *, batch_size=1, target_size=None, max_flow=400, protocol='keras', workers=4,
             per_image=False):
    """Score `model` on `dataset` (a `tf_raft_b200.datasets` FlowDataset without augmentor).

    Runs `model([image1, image2], training=False, last_only=True)` over `dataset.batches(batch_size,
    target_size=target_size, workers=workers)` -- frames crop-or-padded with zeros, padded pixels invalid -- and
    returns the chosen aggregation: {'epe', 'u1', 'u3', 'u5', 'fl_all', 'pixels'}.  per_image=True adds 'records':
    {'counts' (N, 5) [n, <1, <3, <5, outlier], 'sums' (N,) EPE sums} in dataset order.

    Zero padding is what the reference's CropOrPadder does.  Published RAFT numbers pad by edge replication
    (InputPadder), so the two are not directly comparable."""
    if dataset.augmentor is not None:
        raise ValueError('evaluate needs a dataset without aug_params')
    if dataset.is_test:
        raise ValueError('evaluate needs ground truth; this is a test split')
    metrics = FlowMetrics(max_flow=max_flow, protocol=protocol)
    for image1, image2, flow, valid, _ in dataset.batches(batch_size, target_size=target_size, workers=workers,
                                                           device=model.device):
        pred = model([image1, image2], training=False, last_only=True)[-1]
        metrics.update_state(flow, pred, valid)
    counts, sums = metrics.records()
    out = aggregate(counts, sums, metrics.batch_sizes, protocol)
    if per_image:
        out['records'] = {'counts': counts, 'sums': sums}
    return out
