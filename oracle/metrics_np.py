"""NumPy restatement of raft_b200_flow_metrics (include/raft_b200.h): per-image counts [n, epe < 1, epe < 3, epe < 5,
outlier] and the float64 sum of the EPE over the kept pixels.  Every per-pixel step is a separate float32 NumPy
operation, so each is rounded once and none is fused."""
import numpy as np


def pixel_terms(pred, gt, valid=None, max_flow=400):
    """-> (kept mask, epe float32, outlier mask), each (B, H, W)."""
    pred = np.asarray(pred, np.float32)
    gt = np.asarray(gt, np.float32)
    with np.errstate(all='ignore'):
        g0, g1 = gt[..., 0], gt[..., 1]
        mag = np.sqrt(np.add(np.multiply(g0, g0), np.multiply(g1, g1)))
        keep = np.ones(mag.shape, bool) if valid is None else np.asarray(valid, np.float32) != 0
        if max_flow is not None:
            keep &= mag < np.float32(max_flow)
        d0 = np.subtract(pred[..., 0], g0)
        d1 = np.subtract(pred[..., 1], g1)
        epe = np.sqrt(np.add(np.multiply(d0, d0), np.multiply(d1, d1)))
        outlier = (epe > np.float32(3)) & (np.divide(epe, mag) > np.float32(0.05))
    return keep, epe, outlier


def records(pred, gt, valid=None, max_flow=400):
    """-> counts (B, 5) int64, sums (B,) float64."""
    keep, epe, outlier = pixel_terms(pred, gt, valid, max_flow)
    B = keep.shape[0]
    counts = np.zeros((B, 5), np.int64)
    sums = np.zeros(B, np.float64)
    for b in range(B):
        k = keep[b]
        e = epe[b][k]
        counts[b] = [k.sum(), (e < 1).sum(), (e < 3).sum(), (e < 5).sum(), outlier[b][k].sum()]
        sums[b] = np.sum(e.astype(np.float64))
    return counts, sums
