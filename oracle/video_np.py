"""NumPy restatement of RAFT's warm start between the pairs of a video (test infrastructure).

`forward_interpolate` is the fp64 brute force the CUDA kernel (tf_raft_b200/csrc/video.cuh) must match bit for bit.  Per
image of a (B, h, w, 2) float32 flow:
  * source pixel i = y*w + x lands at x1 = x + fx, y1 = y + fy (int64 grid + float32 flow -> float64, one rounding);
  * it is valid iff 0 < x1 < w and 0 < y1 < h (NaN / inf compare false, so they never are);
  * target (X, Y) takes the float32 flow of the valid source minimising d = (x1 - X)**2 + (y1 - Y)**2 in float64, ties
    to the lowest source index (np.argmin returns the first minimum);
  * an image with no valid source gets zero flow (scipy's griddata raises there).
tests/test_video.py checks it against scipy.interpolate.griddata(method='nearest').
"""
import numpy as np


def landing(flow):
    """(x1, y1, valid), each (B, h*w): where every source pixel of a (B, h, w, 2) flow lands, in float64."""
    flow = np.asarray(flow, dtype=np.float32)
    b, h, w, _ = flow.shape
    gy, gx = np.meshgrid(np.arange(h, dtype=np.int64), np.arange(w, dtype=np.int64), indexing='ij')
    x1 = gx.reshape(1, -1) + flow[..., 0].reshape(b, -1)            # int64 + float32 -> float64
    y1 = gy.reshape(1, -1) + flow[..., 1].reshape(b, -1)
    with np.errstate(invalid='ignore'):
        valid = (x1 > 0) & (x1 < w) & (y1 > 0) & (y1 < h)
    return x1, y1, valid


def forward_interpolate(flow, return_index=False):
    """(B, h, w, 2) float32 -> (B, h, w, 2) float32; with return_index also the chosen source index per target
    (B, h*w), -1 where the image has no valid source."""
    flow = np.asarray(flow, dtype=np.float32)
    b, h, w, _ = flow.shape
    n = h * w
    x1, y1, valid = landing(flow)
    tx = np.arange(w, dtype=np.float64)
    out = np.zeros_like(flow).reshape(b, n, 2)
    index = np.full((b, n), -1, dtype=np.int64)
    for k in range(b):
        src = np.nonzero(valid[k])[0]                                 # ascending: argmin's first minimum = lowest index
        if src.size == 0:
            continue
        sx, sy = x1[k, src], y1[k, src]
        dx = sx[None, :] - tx[:, None]                                # (w, sources): the same for every target row
        dx2 = dx * dx
        for Y in range(h):                                            # one target row at a time
            dy = sy - np.float64(Y)
            d = dx2 + (dy * dy)[None, :]
            index[k, Y * w:(Y + 1) * w] = src[np.argmin(d, axis=1)]
        out[k] = flow[k].reshape(n, 2)[index[k]]
    out = out.reshape(b, h, w, 2)
    return (out, index) if return_index else out
