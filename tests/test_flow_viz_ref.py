"""Flow colour wheel on the host: the NumPy restatement (oracle/flow_viz_np.py) against the reference's own output
(tests/golden/flow_viz.npz), the colour wheel, NumPy 2's dtype steps, the PNG writer, and the host-side argument checks
of raft_b200_flow_to_image.  No GPU needed."""
import ctypes
import hashlib
import os
import struct
import zlib

import numpy as np
import pytest
import torch

from oracle import flow_viz_np as F

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'flow_viz.npz')
# Pixels of the golden where the restatement differs from the reference run with NumPy 2.3.5's AVX-512 float32
# arctan2: 5 of 472 710, all one level, all in the 436x1024 case (DESIGN.md section 3.5).
MAX_DIFFERING = 5
EXACT = ('zero_4x6', 'signed_zero_1x6', 'overflow_1x4', 'axis_1x8')


def test_restatement_matches_reference_golden():
    g = np.load(GOLDEN)
    total = differing = 0
    for name, (flow, kw) in F.golden_cases().items():
        img, near = F.flow_to_image(flow, **kw)
        ref = g[name]
        assert img.shape == ref.shape and img.dtype == ref.dtype == np.uint8, name
        d = np.abs(img.astype(np.int16) - ref.astype(np.int16))
        assert d.max() <= 1, (name, int(d.max()))
        differing += int((d.max(-1) > 0).sum())
        total += d.shape[0] * d.shape[1]
        if name in EXACT:
            assert not near.any() and np.array_equal(img, ref), name
    assert total == 472710
    assert differing <= MAX_DIFFERING, differing


def test_edge_cases_known_answers():
    g = np.load(GOLDEN)
    sz = g['signed_zero_1x6'][0]
    assert sz[0].tolist() == [255, 0, 0] and sz[1].tolist() == [255, 0, 43]       # (5, +0) and (5, -0)
    assert (g['zero_4x6'] == 255).all() and (g['overflow_1x4'] == 255).all()      # white: rad = 0 / all normalise to 0
    img, _ = F.flow_to_image(np.zeros((2, 3, 2), np.float32), convert_to_bgr=True)
    assert (img == 255).all()


def test_colorwheel_formulas():
    from tf_raft_b200.datasets import make_colorwheel
    wheel = make_colorwheel()
    assert wheel.shape == (55, 3) and wheel.dtype == np.float64
    np.testing.assert_array_equal(wheel, F.make_colorwheel())
    col = 0
    for (name, n), (c_full, c_ramp, rising) in zip(F.WHEEL_SEGMENTS, [(0, 1, 1), (1, 0, 0), (1, 2, 1), (2, 1, 0),
                                                                      (2, 0, 1), (0, 2, 0)]):
        for j in range(n):
            step = np.floor(255 * j / n)
            assert wheel[col + j, c_full] == 255, name
            assert wheel[col + j, c_ramp] == (step if rising else 255 - step), name
            assert wheel[col + j, 3 - c_full - c_ramp] == 0, name
        col += n
    assert col == 55


def test_nep50_dtype_steps():
    """The dtypes the reference's expressions take under NumPy 2, which the kernels reproduce."""
    assert int(np.__version__.split('.')[0]) >= 2
    u = np.array([[0.5, -3.0]], np.float32)
    v = np.array([[-0.25, 1e-3]], np.float32)
    assert np.clip(u, 0, 5.0).dtype == np.float32
    rad = np.sqrt(np.square(u) + np.square(v))
    assert rad.dtype == np.float32
    assert (u / (np.max(rad) + 1e-5)).dtype == np.float32
    a = np.arctan2(-v, -u) / np.pi
    assert a.dtype == np.float32
    fk = (a + 1) / 2 * 54
    assert fk.dtype == np.float32
    k0 = np.floor(fk).astype(np.int32)
    f = fk - k0
    assert f.dtype == np.float64
    col = (1 - f) * (F.make_colorwheel()[k0, 0] / 255.0)
    assert col.dtype == np.float64 and (1 - rad * (1 - col)).dtype == np.float64
    s = F.steps(u, v)
    for k, dt in (('rad', np.float32), ('a', np.float32), ('fk', np.float32), ('k0', np.int32), ('f', np.float64)):
        assert s[k].dtype == dt, k
    np.testing.assert_array_equal(s['f'], fk - k0)


def test_near_midpoint_mask():
    mid = (np.float64(np.float32(1.0)) + np.float64(np.nextafter(np.float32(1.0), np.float32(2)))) / 2
    x = np.array([1.0, mid, mid * (1 + 2.0 ** -50), mid * (1 + 2.0 ** -40), np.pi])
    assert F.near_midpoint(x).tolist() == [False, True, True, False, False]


def _decode_png(raw):
    pos, chunks = 8, {}
    assert raw[:8] == b'\x89PNG\r\n\x1a\n'
    while pos < len(raw):
        n, kind = struct.unpack('>I4s', raw[pos:pos + 8])
        body = raw[pos + 8:pos + 8 + n]
        assert struct.unpack('>I', raw[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(kind + body) & 0xffffffff
        chunks.setdefault(kind, []).append(body)
        pos += 12 + n
    w, h, depth, ctype, _, _, interlace = struct.unpack('>IIBBBBB', chunks[b'IHDR'][0])
    assert (depth, ctype, interlace) == (8, 2, 0)
    rows = zlib.decompress(b''.join(chunks[b'IDAT']))
    assert len(rows) == h * (1 + 3 * w)
    out = np.frombuffer(rows, np.uint8).reshape(h, 1 + 3 * w)
    assert (out[:, 0] == 0).all()                                           # filter type 0 on every row
    return out[:, 1:].reshape(h, w, 3)


def test_png8_round_trip(tmp_path):
    from tf_raft_b200.datasets import write_png
    img = np.random.default_rng(0).integers(0, 256, (7, 13, 3), dtype=np.uint8)
    write_png(tmp_path / 'a.png', img)
    np.testing.assert_array_equal(_decode_png((tmp_path / 'a.png').read_bytes()), img)
    with pytest.raises(ValueError):
        write_png(tmp_path / 'b.png', img.astype(np.float32))
    try:                                           # cross-check against OpenCV's decoder when it is installed
        import cv2
        np.testing.assert_array_equal(cv2.imread(str(tmp_path / 'a.png'))[:, :, ::-1], img)
    except ImportError:
        pass


def test_write_flow_kitti_bytes_unchanged(tmp_path):
    """The sha256 of write_flow_kitti's file on a fixed input, recorded before it was moved onto write_png."""
    from tf_raft_b200.datasets import write_flow_kitti
    rng = np.random.default_rng(3)
    flow = (rng.integers(-300 * 64, 300 * 64, (6, 11, 2)) / 64.0).astype(np.float32)
    valid = (rng.uniform(size=(6, 11)) > 0.4).astype(np.float32)
    write_flow_kitti(tmp_path / 'k.png', flow, valid)
    write_flow_kitti(tmp_path / 'k2.png', flow)
    digest = [hashlib.sha256((tmp_path / p).read_bytes()).hexdigest() for p in ('k.png', 'k2.png')]
    assert digest == ['7d2d3f2a727b4bc834a33b8ddde1213d8d71ca0ea4e31b776db371e7b76cd3ac',
                      'd38b1050bc31a29bcbd0a399541a650a52683650f913c6e49b39c5204580a24c']


def test_cpu_tensors_are_rejected():
    from tf_raft_b200.datasets import flow_to_image, flow_uv_to_colors
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        flow_to_image(torch.zeros(4, 5, 2))
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        flow_uv_to_colors(torch.zeros(4, 5), torch.zeros(4, 5))


def test_host_side_argument_errors():
    """raft_b200_flow_to_image validates on the host before touching memory (the pointers here are never used)."""
    from tf_raft_b200 import _lib, build
    build.build()
    L = _lib.lib()
    p = ctypes.c_void_p(0x1000)
    call = L.raft_b200_flow_to_image
    assert call(p, p, 2, 1, 4, 4, 1, -1.0, 1, None, 0, p, p, p, None) == -1                # negative clip_flow
    assert call(p, p, 2, 1, 4, 4, 1, float('nan'), 1, None, 0, p, p, p, None) == -1        # NaN clip_flow
    assert call(p, p, 2, 1, 4, 4, 1, float('inf'), 1, None, 0, p, p, p, None) == -1        # inf clip_flow
    assert call(p, p, 3, 1, 4, 4, 0, 0.0, 1, None, 0, p, p, p, None) == -1                 # stride
    assert call(None, p, 2, 1, 4, 4, 0, 0.0, 1, None, 0, p, p, p, None) == -1
    assert call(p, p, 2, 1, 4, 4, 0, 0.0, 1, None, 0, p, None, p, None) == -1              # no work for the reduction
    assert call(p, p, 2, 1, 4, 4, 0, 0.0, 1, None, 0, ctypes.c_void_p(0x1001), p, p, None) == -1   # misaligned image
    assert call(p, p, 2, 0, 4, 4, 0, 0.0, 1, None, 0, p, p, p, None) == -2                 # empty
    assert call(p, p, 2, 1, 0, 4, 0, 0.0, 1, None, 0, p, p, p, None) == -2
    assert call(p, p, 2, 65536, 4, 4, 0, 0.0, 1, None, 0, p, p, p, None) == -2
    assert call(p, p, 2, 1, 65536, 65536, 0, 0.0, 1, None, 0, p, p, p, None) == -2         # H*W >= 2^31
