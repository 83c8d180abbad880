"""Flow file readers / writers -- host-side mirror of tf_raft/datasets/frame_utils.py:12-68, 83-107, 123-137 (NumPy,
and PIL for frames; the evaluation scripts feed `RAFT.test_step` with what these return).

.flo (Middlebury): float32 tag 202021.25, int32 width, int32 height, then height x width x (u, v) float32, little endian.
KITTI flow PNG: 16-bit RGB, u = (R - 2^15) / 64, v = (G - 2^15) / 64, B = valid flag.
`write_png` writes the 8- and 16-bit RGB PNGs (KITTI flows, VisFlowCallback's pictures) without an image library.
"""
import os
import re
import struct
import zlib

import numpy as np

TAG_FLOAT = 202021.25


def read_flow(path):
    """frame_utils.py:12-31 readFlow -> (H, W, 2) float32.  Raises on a wrong tag (the reference prints and returns None)."""
    with open(path, 'rb') as f:
        head = f.read(12)
        if len(head) < 12 or struct.unpack('<f', head[:4])[0] != TAG_FLOAT:
            raise ValueError(f'{path}: magic number incorrect, not a .flo file')
        w, h = struct.unpack('<ii', head[4:])
        data = np.frombuffer(f.read(8 * w * h), dtype='<f4')
    if data.size != 2 * w * h:
        raise ValueError(f'{path}: truncated .flo file ({data.size} of {2 * w * h} values)')
    return data.reshape(h, w, 2).astype(np.float32)


def write_flow(path, flow):
    """frame_utils.py:70-99 writeFlow: (H, W, 2) -> .flo."""
    flow = np.asarray(flow, dtype=np.float32)
    if flow.ndim != 3 or flow.shape[2] != 2:
        raise ValueError('flow must be (H, W, 2)')
    h, w, _ = flow.shape
    with open(path, 'wb') as f:
        f.write(struct.pack('<fii', TAG_FLOAT, w, h))
        f.write(np.ascontiguousarray(flow, dtype='<f4').tobytes())


def _png_chunks(data):
    if data[:8] != b'\x89PNG\r\n\x1a\n':
        raise ValueError('not a PNG file')
    pos = 8
    while pos < len(data):
        n, kind = struct.unpack('>I4s', data[pos:pos + 8])
        yield kind, data[pos + 8:pos + 8 + n]
        pos += 12 + n


def _read_png16_rgb(path):
    """Minimal decoder for the non-interlaced 16-bit RGB PNGs of KITTI (cv2.IMREAD_ANYDEPTH equivalent, no OpenCV needed)."""
    raw = open(path, 'rb').read()
    ihdr, idat = None, []
    for kind, body in _png_chunks(raw):
        if kind == b'IHDR':
            ihdr = struct.unpack('>IIBBBBB', body)
        elif kind == b'IDAT':
            idat.append(body)
    w, h, depth, ctype, _, _, interlace = ihdr
    if depth != 16 or ctype != 2 or interlace != 0:
        raise ValueError(f'{path}: expected a non-interlaced 16-bit RGB PNG (KITTI flow), got depth {depth} colour type {ctype}')
    rows = zlib.decompress(b''.join(idat))
    bpp, stride = 6, 6 * w
    out = np.zeros((h, stride), dtype=np.uint8)
    prev = np.zeros(stride, dtype=np.int32)
    pos = 0
    for y in range(h):
        ft = rows[pos]
        line = np.frombuffer(rows, dtype=np.uint8, count=stride, offset=pos + 1).astype(np.int32)
        pos += stride + 1
        if ft == 0:
            cur = line
        elif ft == 2:
            cur = (line + prev) & 255
        else:                                        # Sub / Average / Paeth need the running left neighbour
            cur = np.zeros(stride, dtype=np.int32)
            for i in range(stride):
                a = cur[i - bpp] if i >= bpp else 0
                b = prev[i]
                c = prev[i - bpp] if i >= bpp else 0
                if ft == 1:
                    pred = a
                elif ft == 3:
                    pred = (a + b) >> 1
                else:
                    pa, pb, pc = abs(b - c), abs(a - c), abs(a + b - 2 * c)
                    pred = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
                cur[i] = (line[i] + pred) & 255
        out[y] = cur
        prev = cur
    return out.reshape(h, w, 3, 2).astype(np.uint16) @ np.array([256, 1], dtype=np.uint16)


def inflate_png16(path):
    """The host half of a KITTI flow PNG read: chunks parsed, IDATs joined and inflated -> (filtered scanlines (bytes),
    h, w).  The rows are checked for length and filter bytes 0-4 here; `read_flow_kitti_batch` undoes the filters on
    the GPU.  Raises ValueError naming the file for anything but a well-formed non-interlaced 16-bit RGB PNG."""
    try:
        raw = open(path, 'rb').read()
        ihdr, idat = None, []
        for kind, body in _png_chunks(raw):
            if kind == b'IHDR':
                ihdr = struct.unpack('>IIBBBBB', body)
            elif kind == b'IDAT':
                idat.append(body)
        if ihdr is None:
            raise ValueError('no IHDR chunk')
        w, h, depth, ctype, _, _, interlace = ihdr
        if depth != 16 or ctype != 2 or interlace != 0:
            raise ValueError(f'expected a non-interlaced 16-bit RGB PNG (KITTI flow), got depth {depth} colour type '
                             f'{ctype} interlace {interlace}')
        rows = zlib.decompress(b''.join(idat))
    except (struct.error, zlib.error, ValueError) as e:
        raise ValueError(f'{path}: {e}') from None
    if h < 1 or w < 1 or len(rows) != h * (1 + 6 * w):
        raise ValueError(f'{path}: {len(rows)} bytes of scanlines, expected {h} x (1 + 6 x {w})')
    filters = np.frombuffer(rows, dtype=np.uint8)[::1 + 6 * w]
    if filters.max() > 4:
        raise ValueError(f'{path}: unknown PNG filter type {int(filters.max())} in row {int(np.argmax(filters > 4))}')
    return rows, h, w


def read_pfm(path):
    """frame_utils.py:33-68 readPFM: 'PF' (3 channels) or 'Pf' (1), width and height, then a scale whose sign gives the
    byte order (negative: little endian); rows are stored bottom-up, so the array is flipped.  -> float32 (H, W[, 3])."""
    with open(path, 'rb') as f:
        header = f.readline().rstrip()
        if header not in (b'PF', b'Pf'):
            raise ValueError(f'{path}: not a PFM file')
        dims = re.match(rb'^(\d+)\s(\d+)\s$', f.readline())
        if not dims:
            raise ValueError(f'{path}: malformed PFM header')
        width, height = map(int, dims.groups())
        scale = float(f.readline().rstrip())
        data = np.fromfile(f, ('<' if scale < 0 else '>') + 'f')
    shape = (height, width, 3) if header == b'PF' else (height, width)
    return np.flipud(np.reshape(data, shape))


def read_gen(path, pil=False):
    """frame_utils.py:123-137 read_gen: dispatch on the extension.  .png / .jpeg / .ppm / .jpg -> PIL.Image (opened
    lazily, as the reference); .bin / .raw -> np.load; .flo -> read_flow; .pfm -> read_pfm as float32, a colour PFM
    without its last channel; anything else -> [].  `pil` is accepted and ignored, as in the reference."""
    ext = os.path.splitext(path)[-1]
    if ext in ('.png', '.jpeg', '.ppm', '.jpg'):
        from PIL import Image
        return Image.open(path)
    if ext in ('.bin', '.raw'):
        return np.load(path)
    if ext == '.flo':
        return read_flow(path).astype(np.float32)
    if ext == '.pfm':
        flow = read_pfm(path).astype(np.float32)
        return flow if flow.ndim == 2 else flow[:, :, :-1]
    return []


def read_flow_kitti(path):
    """frame_utils.py:102-107 readFlowKITTI -> (flow (H, W, 2) float32, valid (H, W) float32)."""
    rgb = _read_png16_rgb(path).astype(np.float32)
    flow = (rgb[:, :, :2] - 2 ** 15) / 64.0
    return flow.astype(np.float32), rgb[:, :, 2]


def write_flow_kitti(path, flow, valid=None):
    """frame_utils.py:116-120 writeFlowKITTI: 16-bit RGB PNG (filter type 0 rows)."""
    flow = np.asarray(flow, dtype=np.float32)
    h, w, _ = flow.shape
    valid = np.ones((h, w), np.float32) if valid is None else np.asarray(valid, np.float32)
    write_png(path, np.concatenate([64.0 * flow + 2 ** 15, valid[..., None]], axis=-1).astype(np.uint16))


def write_png(path, image):
    """Non-interlaced RGB PNG of an (H, W, 3) uint8 (8-bit) or uint16 (16-bit) array: filter type 0 rows, one zlib
    IDAT chunk.  No image library needed."""
    image = np.asarray(image)
    if image.ndim != 3 or image.shape[2] != 3 or image.dtype not in (np.uint8, np.uint16):
        raise ValueError(f'write_png: expected an (H, W, 3) uint8 or uint16 array, got {image.shape} {image.dtype}')
    h, w, _ = image.shape
    depth = 8 * image.dtype.itemsize
    be = image.astype('>u2' if depth == 16 else np.uint8).tobytes()
    stride = 3 * image.dtype.itemsize * w
    rows = b''.join(b'\x00' + be[y * stride:(y + 1) * stride] for y in range(h))

    def chunk(kind, body):
        return struct.pack('>I', len(body)) + kind + body + struct.pack('>I', zlib.crc32(kind + body) & 0xffffffff)
    with open(path, 'wb') as f:
        f.write(b'\x89PNG\r\n\x1a\n' + chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, depth, 2, 0, 0, 0)) +
                chunk(b'IDAT', zlib.compress(rows)) + chunk(b'IEND', b''))
