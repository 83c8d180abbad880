"""The data-path kernels at HD1K (1080x2560) and multi-megapixel sizes, against independent host references.

- png16_decode_kernel: row widths that give every Sub run length (ceil(W / 256) pixels per thread) up to the width
  limit, every W mod 8 tail of the Average / Paeth chains, planted Paeth ties and Average wraps, a mixed-size launch
  with one file far wider than the rest, and files from real writers -- each bit for bit against the NumPy reader
  (`read_flow_kitti`) and, where it imports, OpenCV's libpng reader.  Width 16385 is refused on the host.
- flow_metrics_*_kernel: images of more than 256 CTA partials (kMetChunk = 8192 pixels each), so the final kernel's
  loop takes a second pass, against oracle/metrics_np.py and an exactly rounded sum (math.fsum).
- augment_*_kernel (sparse): HD1K's scale range, KITTI and HD1K in one launch, and the training loader on a
  `2 * kitti + hd1k` tree, bit for bit against oracle/augment_np.py and `augmentor.batch`.
- pad_planes_kernel at 1080x2560 and in a batch mixing KITTI and HD1K items, against np.pad; `evaluate` on 1080x2560
  items against RAFT's pad / predict / unpad / score recipe.

The unmarked tests are host-only checks: they pin the NumPy reader to libpng on the planted files and show that the
sizes and seeds below reach the branches named above.
"""
import math
import os
import random
import re

import numpy as np
import pytest
import torch

from oracle import metrics_np, weights
from tf_raft_b200.datasets import frame_utils
from test_gpu_augment import _check as _check_augment, _sample
from test_gpu_eval import FILTERS, _check as _check_metrics, _decode_files, _expected, _random_case, _records, \
    _rgb16, encode_png16
from test_gpu_pad import _np_pad, _planes, _same

F32 = np.float32
HD1K = (1080, 2560)
KITTI_SIZES = [(375, 1242), (370, 1226)]

PNG_THREADS = 256                      # kPngThreads (csrc/dataset.cuh): Sub gives each thread ceil(W / 256) pixels
PNG_MAX_WIDTH = 16384                  # kPngMaxWidth
MET_CHUNK = 8192                       # kMetChunk: pixels per CTA partial of the metrics kernel
ERR_BAD_SHAPE = -2                     # RAFT_ERR_BAD_SHAPE (include/raft_b200.h)

WIDTHS = [255, 256, 257, 511, 512, 513] + [2560 + r for r in range(8)] + [PNG_MAX_WIDTH]
METRIC_SHAPES = [(3, 1024, 2048), (3, 3, 699051), (3, 1080, 2560), (3, 1088, 2560), (1, 2160, 3840)]

# The HD1K stage of the reference's Sintel mixture (tf_raft/datasets/dataset.py:292-293), at its 368x768 crop.
CROP = (368, 768)
HD1K_AUG = {'crop_size': CROP, 'min_scale': -0.5, 'max_scale': 0.2, 'do_flip': True}
KITTI_AUG = {'crop_size': CROP, 'min_scale': -0.3, 'max_scale': 0.5, 'do_flip': True}
HD1K_SEED, HD1K_FULL = 22, (1, 5)      # six draws; the samples at HD1K_FULL get a fully valid map
MIXED_SEED = 127
MIXED_SHAPES = [HD1K, KITTI_SIZES[0], HD1K, KITTI_SIZES[1], KITTI_SIZES[0]]


def _cv2():
    try:
        import cv2
        return cv2
    except ImportError:
        return None


def _cv2_read(cv2, path):
    """cv2.imread(IMREAD_UNCHANGED) (libpng), BGR reversed, as read_flow_kitti's (flow, valid)."""
    bgr = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    assert bgr is not None and bgr.dtype == np.uint16, path
    return _expected(bgr[..., ::-1])


def _assert_same_decode(got, want, what):
    np.testing.assert_array_equal(got[0], want[0], err_msg=what)
    np.testing.assert_array_equal(got[1], want[1], err_msg=what)
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes(), what


# --------------------------------------------------------------------------------------------- planted PNG rows
def _planted_rgb(h, w, seed):
    """(h, w, 3) uint16 whose bytes make every Paeth tie and Average's odd and wrapping sums common.  Rows cycle
    through: one byte value twice (a = b = c); bytes from a small evenly spaced set, then that row moved one pixel
    left (left = above, so pa = pb); then two rows of bytes near 0 and 255 (odd sums at both ends, wraps)."""
    rng = np.random.default_rng(seed)
    rows = np.empty((h, 6 * w), np.uint8)
    for y in range(h):
        kind = y % 6
        if kind == 0:
            rows[y] = rng.integers(0, 256)
        elif kind in (1, 3):
            rows[y] = np.concatenate([rows[y - 1, 6:], rng.integers(0, 256, 6)]) if kind == 3 else rows[y - 1]
        elif kind == 2:
            rows[y] = rng.choice([40, 60, 80, 100, 120], 6 * w)
        else:
            rows[y] = rng.choice([0, 1, 2, 253, 254, 255], 6 * w)
    return rows.reshape(h, w, 3, 2).astype(np.uint16) @ np.array([256, 1], np.uint16)


def _filter_terms(rgb):
    """Per byte of every row but the first: (a, b, c, x) = left, above, above-left and the byte itself, bpp 6."""
    h, w, _ = rgb.shape
    x = rgb.astype('>u2').view(np.uint8).reshape(h, 6 * w).astype(np.int64)
    left = np.concatenate([np.zeros((h, 6), np.int64), x[:, :-6]], axis=1)
    a, b, c = left[1:], x[:-1], left[:-1]
    return a, b, c, x[1:]


def _tie_counts(rgb):
    """How often each Paeth tie and each Average case occurs in the rows of `rgb` (rows after the first)."""
    a, b, c, x = _filter_terms(rgb)
    pa, pb, pc = np.abs(b - c), np.abs(a - c), np.abs(a + b - 2 * c)
    avg = (a + b) >> 1
    odd = (a + b) % 2 == 1
    return {'pa=pb=pc': int(((pa == pb) & (pb == pc)).sum()), 'pa=pb<pc': int(((pa == pb) & (pa < pc)).sum()),
            'pb=pc<pa': int(((pb == pc) & (pb < pa)).sum()), 'pa=pc<pb': int(((pa == pc) & (pa < pb)).sum()),
            'avg odd near 0': int((odd & (a + b < 8)).sum()), 'avg odd near 510': int((odd & (a + b > 502)).sum()),
            'avg wraps': int(((x - avg) % 256 + avg > 255).sum())}


PLANTED = [((12, 2560), [4]), ((12, 2560), [3]), ((12, 13), [4, 3]), ((9, 2563), [0, 1, 2, 3, 4, 4, 3, 1, 2])]


def _write_planted(root):
    paths, counts = [], []
    for k, ((h, w), filters) in enumerate(PLANTED):
        rgb = _planted_rgb(h, w, 40 + k)
        p = os.path.join(str(root), f'planted{k}_{h}x{w}.png')
        encode_png16(p, rgb, filters, n_idat=1 + k % 3)
        paths.append(p)
        counts.append(_tie_counts(rgb))
    return paths, counts


def test_planted_png_files_reach_every_tie_and_the_numpy_reader_equals_libpng(tmp_path):
    """Host only: the planted files hold every Paeth tie and Average's odd and wrapping sums, and on them the NumPy
    reader (the GPU tests' oracle) equals OpenCV's libpng reader."""
    paths, counts = _write_planted(tmp_path)
    paeth = counts[0]                                             # the file with Paeth on every row
    for kind in ('pa=pb=pc', 'pa=pb<pc', 'pb=pc<pa', 'pa=pc<pb'):
        assert paeth[kind] > 0, (kind, paeth)
    for kind in ('avg odd near 0', 'avg odd near 510', 'avg wraps'):
        assert counts[1][kind] > 0, (kind, counts[1])
    cv2 = _cv2()
    if cv2 is None:
        pytest.skip('cv2 is not installed')
    for p in paths:
        _assert_same_decode(frame_utils.read_flow_kitti(p), _cv2_read(cv2, p), p)


def test_sizes_and_seeds_reach_the_branches():
    """Host only: the widths give Sub runs of 1, 2, 3, 10 and 64 pixels and every W mod 8 chain tail; the metrics
    shapes give 256, 257 and more than 256 partials; the seeded draws give an HD1K sample at a scale of 0.75 or below
    and KITTI samples at the (crop + 1) / size clip, which HD1K never reaches at this crop."""
    runs = {-(-w // PNG_THREADS) for w in WIDTHS}
    assert {1, 2, 3, 10, 64} <= runs and {w % 8 for w in WIDTHS} == set(range(8))
    chunks = [-(-h * w // MET_CHUNK) for _, h, w in METRIC_SHAPES]
    assert chunks == [256, 257, 338, 340, 1013]
    hd1k, mixed = _hd1k_draws(), _mixed_draws()
    assert any(p.spatial and p.scale_x <= 0.75 for p in hd1k)
    assert all(hd1k[i].spatial and hd1k[i].scale_x <= 0.75 for i in HD1K_FULL)
    assert any(p.hflip for p in hd1k) and any(not p.spatial for p in hd1k)
    clip = [max((CROP[0] + 1) / h, (CROP[1] + 1) / w) for h, w in MIXED_SHAPES]
    assert max(clip[0], clip[2]) < 0.35
    at_clip = [s != HD1K and p.spatial and p.scale_x == c for s, p, c in zip(MIXED_SHAPES, mixed, clip)]
    assert sum(at_clip) >= 2
    assert any(p.spatial and p.scale_x < 0.75 for s, p in zip(MIXED_SHAPES, mixed) if s == HD1K)


# --------------------------------------------------------------------------------------------- PNG decoder
@pytest.mark.gpu
def test_png_decoder_row_widths(tmp_path):
    """Widths 255-513, 2560 + 0..7 and 16384, each filter on every row and the mixed cycle, all in one launch (so the
    16384-wide files set every CTA's row buffers): equal to the NumPy reader and to libpng, bit for bit."""
    cv2 = _cv2()
    paths = []
    for w in WIDTHS:
        h = 3 if w == PNG_MAX_WIDTH else 5
        for name, filters in FILTERS.items():
            p = str(tmp_path / f'{name}_{h}x{w}.png')
            encode_png16(p, _rgb16(h, w, w + 7 * len(paths)), filters, n_idat=1 + len(paths) % 3)
            paths.append(p)
    for p, got in zip(paths, _decode_files(paths)):
        _assert_same_decode(got, frame_utils.read_flow_kitti(p), p)
        if cv2 is not None:
            _assert_same_decode(got, _cv2_read(cv2, p), p)


@pytest.mark.gpu
def test_png_decoder_planted_ties(tmp_path):
    paths, _ = _write_planted(tmp_path)
    for p, got in zip(paths, _decode_files(paths)):
        _assert_same_decode(got, frame_utils.read_flow_kitti(p), p)


@pytest.mark.gpu
def test_png_decoder_mixed_batch_with_hd1k(tmp_path):
    """1080x2560 (the mixed filter cycle), 375x1242 and 2x3 in one launch, whose row buffers the HD1K file sizes; the
    same files in the reverse order give the same bytes.  The HD1K file is checked against the values it encodes
    (which the NumPy reader returns for every filter, test_png_decoder_row_widths) and libpng, the others against the
    NumPy reader."""
    cv2 = _cv2()
    specs = [(HD1K, FILTERS['mixed']), ((375, 1242), [2, 4, 0, 3, 1]), ((2, 3), [3, 4])]
    paths, rgbs = [], []
    for k, ((h, w), filters) in enumerate(specs):
        rgb = _rgb16(h, w, 60 + k)
        p = str(tmp_path / f'mixed{k}_{h}x{w}.png')
        encode_png16(p, rgb, filters)
        paths.append(p)
        rgbs.append(rgb)
    got = _decode_files(paths)
    _assert_same_decode(got[0], _expected(rgbs[0]), paths[0])
    if cv2 is not None:
        _assert_same_decode(got[0], _cv2_read(cv2, paths[0]), paths[0])
    for p, g in zip(paths[1:], got[1:]):
        _assert_same_decode(g, frame_utils.read_flow_kitti(p), p)
    back = _decode_files(paths[::-1])[::-1]
    for p, g, b in zip(paths, got, back):
        _assert_same_decode(b, g, p + ' (reverse order)')


@pytest.mark.gpu
def test_png_decoder_hd1k_files_from_real_writers(tmp_path):
    """A 1080x2560 file from write_flow_kitti (None rows) and one from cv2.imwrite, whose rows libpng filters."""
    from tf_raft_b200.datasets import read_flow_kitti_batch
    rng = np.random.default_rng(4)
    paths, want = [], []
    p = str(tmp_path / 'written.png')
    frame_utils.write_flow_kitti(p, rng.normal(0, 30, HD1K + (2,)).astype(F32), (rng.random(HD1K) < 0.5).astype(F32))
    paths.append(p)
    want.append(frame_utils.read_flow_kitti(p))
    cv2 = _cv2()
    if cv2 is not None:
        p = str(tmp_path / 'cv2.png')
        rgb = np.clip(64 * rng.normal(0, 30, HD1K + (3,)) + 2 ** 15, 0, 65535).astype(np.uint16)
        rgb[..., 2] = rng.integers(0, 2, HD1K)
        assert cv2.imwrite(p, rgb[..., ::-1])
        rows, h, w = frame_utils.inflate_png16(p)
        print('cv2.imwrite filter types:', sorted(set(np.frombuffer(rows, np.uint8)[::1 + 6 * w].tolist())))
        paths.append(p)
        want.append(_expected(rgb))
        _assert_same_decode(_cv2_read(cv2, p), want[-1], p)
    flow, valid = read_flow_kitti_batch(paths)
    for i, (p, w) in enumerate(zip(paths, want)):
        _assert_same_decode((flow[i].cpu().numpy(), valid[i].cpu().numpy()), w, p)


@pytest.mark.gpu
def test_png_decoder_refuses_width_past_the_limit(tmp_path):
    """Width 16385 is refused by the host check with the library's 'bad shape' error and never launches; 16384 in the
    same buffer decodes."""
    from tf_raft_b200 import _lib
    from tf_raft_b200.datasets import read_flow_kitti_batch
    from tf_raft_b200.datasets.png16 import decode_png16
    w = PNG_MAX_WIDTH + 1
    data = torch.zeros(2 * (1 + 6 * w), dtype=torch.uint8, device='cuda')
    text = re.escape(f'png16_flow_decode failed: [{ERR_BAD_SHAPE}] {_lib.strerror(ERR_BAD_SHAPE)}')
    _lib.launch_count_reset()
    with pytest.raises(RuntimeError, match=text):
        decode_png16(data, [(0, 2, w)], ['wide.png'])
    with pytest.raises(RuntimeError, match=text):                # a narrow file in the batch does not help
        decode_png16(data, [(0, 1, 3), (0, 1, w)], ['narrow.png', 'wide.png'])
    p = str(tmp_path / 'wide.png')
    frame_utils.write_flow_kitti(p, np.zeros((1, w, 2), F32))
    with pytest.raises(RuntimeError, match=text):
        read_flow_kitti_batch([p])
    assert _lib.launch_count() == 0
    flow, valid = decode_png16(data, [(0, 2, PNG_MAX_WIDTH)], ['limit.png'])[0]
    assert _lib.launch_count() == 1
    assert bool((flow == -512).all()) and bool((valid == 0).all())     # zero bytes: (0 - 2^15) / 64


# --------------------------------------------------------------------------------------------- metrics
def _fsum_check(pred, gt, valid, sums):
    """Each image's sum against math.fsum of its float32 EPEs (exactly rounded), within n * 2^-53 of the sum of
    |EPE|: the bound on n fp64 additions of non-negative terms in any order.  A partial dropped or added twice moves
    the sum by thousands of EPEs."""
    keep, epe, _ = metrics_np.pixel_terms(pred, gt, valid)
    for b in range(len(sums)):
        e = epe[b][keep[b]].astype(np.float64)
        exact = math.fsum(e)
        assert abs(sums[b] - exact) <= e.size * 2.0 ** -53 * exact, (b, sums[b], exact)


@pytest.mark.gpu
@pytest.mark.parametrize('shape', METRIC_SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_metrics_past_256_partials(shape):
    """256, 257, 338, 340 and 1013 partials per image: against the NumPy oracle (counts exact, sums to 1e-12), against
    fsum, and each image's record bit-identical alone and in the batch."""
    B, H, W = shape
    pred, gt, valid = _random_case(B, H, W, seed=H + W)
    c, s = _check_metrics(pred, gt, valid)
    _fsum_check(pred, gt, valid, s)
    for b in range(B):
        c1, s1 = _records(pred[b:b + 1], gt[b:b + 1], valid[b:b + 1])
        np.testing.assert_array_equal(c1[0], c[b])
        assert s1[0].tobytes() == s[b].tobytes(), b


@pytest.mark.gpu
def test_metrics_planted_pixels_in_boundary_partials():
    """1088x2560 (340 partials).  Image 0 is the base; image 1 has, in each of partials 0, 255, 256 and 339, one
    outlier and one invalid pixel; images 2-5 each have one NaN EPE in one of those partials.  The planted pixels start
    as exact matches (EPE 0), so the counts move by exactly them, and a NaN makes the image's sum NaN."""
    H, W = 1088, 2560
    nchunk = -(-H * W // MET_CHUNK)
    parts = [0, 255, 256, nchunk - 1]
    pred, gt, valid = _random_case(1, H, W, seed=77)
    pred, gt, valid = (np.repeat(x, 6, axis=0) for x in (pred, gt, valid))
    pf, gf, vf = pred.reshape(6, -1, 2), gt.reshape(6, -1, 2), valid.reshape(6, -1)
    spots = {k: [k * MET_CHUNK + 1234 + d for d in (0, 1, 2)] for k in parts}
    for k in parts:
        last = min((k + 1) * MET_CHUNK, H * W) - 1
        spots[k][2] = last                                        # the last pixel of the partial
        for i in spots[k]:
            gf[:, i] = (1.0, 0.0)
            pf[:, i] = (1.0, 0.0)
            vf[:, i] = 1.0
    for k in parts:
        out, inv, nan = spots[k]
        pf[1, out] = (11.0, 0.0)                                  # epe 10 > 3 and > 5% of |gt| = 1
        vf[1, inv] = 0.0
    for j, k in enumerate(parts):
        pf[2 + j, spots[k][2]] = (np.nan, 0.0)
    c, s = _check_metrics(pred, gt, valid)
    _fsum_check(pred[:2], gt[:2], valid[:2], s[:2])
    n = len(parts)
    np.testing.assert_array_equal(c[1] - c[0], [-n, -2 * n, -2 * n, -2 * n, n])
    for j in range(n):
        np.testing.assert_array_equal(c[2 + j] - c[0], [0, -1, -1, -1, 0])
        assert np.isnan(s[2 + j]), parts[j]
    assert np.isfinite(s[:2]).all()


# --------------------------------------------------------------------------------------------- sparse augmentation
def _sparse_aug(params=HD1K_AUG):
    from tf_raft_b200.datasets import SparseFlowAugmentor
    return SparseFlowAugmentor(**params)


def _hd1k_draws():
    aug = _sparse_aug()
    np.random.seed(HD1K_SEED)
    random.seed(HD1K_SEED)
    return [aug.sample_params(*HD1K) for _ in range(6)]


def _mixed_draws():
    aug = _sparse_aug()
    np.random.seed(MIXED_SEED)
    random.seed(MIXED_SEED)
    return [aug.sample_params(*s) for s in MIXED_SHAPES]


@pytest.mark.gpu
def test_sparse_augment_hd1k_seeded(tmp_path):
    """Six seeded HD1K draws on 1080x2560 sources, two launches of three: valid density 0.35, and fully valid maps at
    scales near 2^-0.5, where about half the sources land on a target another source also hits."""
    aug = _sparse_aug()
    params = _hd1k_draws()
    rng = np.random.default_rng(HD1K_SEED)
    samples = [_sample(rng, *HD1K, sparse=True, density=1.01 if i in HD1K_FULL else 0.35) for i in range(6)]
    for k in (0, 3):
        got = _check_augment(aug, samples[k:k + 3], params[k:k + 3], True)
        for j in range(3):
            if k + j in HD1K_FULL:
                assert got[3][j].mean() > 0.4                     # most targets of a dense map stay valid


@pytest.mark.gpu
def test_sparse_augment_mixed_kitti_hd1k_launch():
    """HD1K, KITTI 375x1242, HD1K, KITTI 370x1226, KITTI 375x1242 in one sparse launch, each with its own workspace
    offset and target map: equal to the per-sample calls and to the oracle."""
    aug = _sparse_aug()
    params = _mixed_draws()
    rng = np.random.default_rng(MIXED_SEED)
    samples = [_sample(rng, *s, sparse=True, density=1.01 if k == 2 else 0.3) for k, s in enumerate(MIXED_SHAPES)]
    got = _check_augment(aug, samples, params, True)
    for i, (s, p) in enumerate(zip(samples, params)):
        one = aug(*(torch.from_numpy(a).cuda() for a in s), params=p)
        for k in range(4):
            assert torch.equal(one[k].cpu(), torch.from_numpy(got[k][i])), (i, k)


# --------------------------------------------------------------------------------------------- a synthetic tree
def _write_tree(root, seed=0):
    """KITTI training (375x1242 and 370x1226 pairs) and one HD1K sequence of three 1080x2560 frames, frames by
    write_png and flow PNGs by write_flow_kitti."""
    rng = np.random.default_rng(seed)

    def frame(h, w):
        base = rng.integers(0, 256, (h // 6 + 2, w // 6 + 2, 3)).astype(np.uint8)
        return np.kron(base, np.ones((6, 6, 1), np.uint8))[:h, :w]

    def flow_png(path, h, w):
        frame_utils.write_flow_kitti(path, rng.normal(0, 20, (h, w, 2)).astype(F32),
                                     (rng.random((h, w)) < 0.4).astype(F32))

    d = os.path.join(root, 'kitti', 'training')
    for sub in ('image_2', 'flow_occ'):
        os.makedirs(os.path.join(d, sub))
    for i, (h, w) in enumerate(KITTI_SIZES):
        for t in (10, 11):
            frame_utils.write_png(os.path.join(d, 'image_2', '%06d_%d.png' % (i, t)), frame(h, w))
        flow_png(os.path.join(d, 'flow_occ', '%06d_10.png' % i), h, w)
    for sub in ('hd1k_input/image_2', 'hd1k_flow_gt/flow_occ'):
        os.makedirs(os.path.join(root, 'hd1k', sub))
    for i in range(3):
        frame_utils.write_png(os.path.join(root, 'hd1k', 'hd1k_input', 'image_2', '000000_%04d.png' % i), frame(*HD1K))
        flow_png(os.path.join(root, 'hd1k', 'hd1k_flow_gt', 'flow_occ', '000000_%04d.png' % i), *HD1K)


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('hd1k'))
    _write_tree(root)
    return root


def _datasets(root, kitti_aug=None, hd1k_aug=None):
    from tf_raft_b200 import datasets as D
    return D.KITTI(kitti_aug, root=os.path.join(root, 'kitti')), D.HD1K(hd1k_aug, root=os.path.join(root, 'hd1k'))


@pytest.mark.gpu
def test_training_loader_kitti_hd1k_mixture(tree):
    """`2 * kitti + hd1k` through FlowDataset.batches in training mode equals augmentor.batch on the same items under
    the same seeds.  `+` keeps the left operand's augmentor, as the reference's does, so the HD1K items take KITTI's
    draws; the second batch mixes KITTI and HD1K items, and the HD1K flow PNGs are decoded on the GPU."""
    kitti, hd1k = _datasets(tree, KITTI_AUG, HD1K_AUG)
    ds = 2 * kitti + hd1k
    plain_k, plain_h = _datasets(tree)
    plain = 2 * plain_k + plain_h
    assert len(ds) == len(plain) == 6 and ds.sparse
    np.random.seed(9)
    random.seed(9)
    got = [tuple(t.cpu() for t in b) for b in ds.batches(3, workers=3)]
    np.random.seed(9)
    random.seed(9)
    items = [plain[i] for i in range(len(plain))]
    assert [it[0].shape[:2] for it in items] == KITTI_SIZES * 2 + [HD1K] * 2
    want = [tuple(t.cpu() for t in ds.augmentor.batch(items[k:k + 3])) for k in (0, 3)]
    assert len(got) == len(want) == 2
    for g, w in zip(got, want):
        for a, b in zip(g, w):
            assert torch.equal(a, b)


# --------------------------------------------------------------------------------------------- padding
@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['sintel', 'kitti'])
def test_pad_kernel_at_hd1k_size(mode):
    """HD1K frames are 1080x2560, both multiples of 8, so InputPadder hands them back untouched without a launch.  The
    pad kernel itself at that size: two items' 1080x2560 frames, flows (NaN, -0.0 and inf in them) and valid maps into
    1088x2568 at the mode's placement, edge and zero fill, in one launch, against np.pad bit for bit."""
    from tf_raft_b200 import InputPadder, _lib
    from tf_raft_b200.preprocess import REPLICATE, ZERO, pad_planes, placement
    planes = [_planes(*HD1K, seed) for seed in (1, 2)]
    img = torch.from_numpy(np.stack([p[0] for p in planes])).cuda()
    flow = torch.from_numpy(np.stack([p[1] for p in planes])).cuda()
    padder = InputPadder(img.shape, mode)
    _lib.launch_count_reset()
    a, b = padder.pad(img, flow)
    assert _lib.launch_count() == 0 and a is img and b is flow and padder.padded_size == HD1K
    (h, w), (H, W) = HD1K, (1088, 2568)
    top, left = placement(h, w, H, W, mode)
    jobs, want = [], []
    for fill in (REPLICATE, ZERO):
        for x in (x for item in planes for x in item):
            src = torch.from_numpy(x).cuda()
            jobs.append((src, torch.full((H, W) + x.shape[2:], 77, dtype=src.dtype, device='cuda'), top, left, fill))
            want.append(_np_pad(x, top, H - h - top, left, W - w - left, fill == REPLICATE))
    _lib.launch_count_reset()
    pad_planes(jobs)
    assert _lib.launch_count() == 1
    for (_, dst, *_, fill), x in zip(jobs, want):
        assert _same(dst, x), (mode, fill, x.dtype, x.shape)


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['sintel', 'kitti'])
def test_loader_replicate_batch_mixes_kitti_and_hd1k(tree, mode):
    """KITTI and HD1K items in one 1088x2560 batch of FlowDataset.batches(padding='replicate'): frames edge-padded,
    flow and valid zero-padded, each at its own placement, against np.pad bit for bit."""
    from tf_raft_b200.preprocess import placement
    kitti, hd1k = _datasets(tree)
    ds = kitti + hd1k
    H, W = 1088, 2560
    (img1, img2, flow, valid, sizes), = list(ds.batches(4, target_size=(H, W), padding='replicate', pad_mode=mode,
                                                        workers=2))
    assert sizes == KITTI_SIZES + [HD1K] * 2
    for k, (h, w) in enumerate(sizes):
        a, b, f, v = ds[k]
        top, left = placement(h, w, H, W, mode)
        pads = (top, H - h - top, left, W - w - left)
        assert _same(img1[k], _np_pad(a, *pads, True)) and _same(img2[k], _np_pad(b, *pads, True)), (k, mode)
        assert _same(flow[k], _np_pad(f, *pads, False)) and _same(valid[k], _np_pad(np.asarray(v, F32), *pads, False))


# --------------------------------------------------------------------------------------------- evaluate
@pytest.mark.gpu
def test_evaluate_hd1k_items(tree):
    """`evaluate(padding='replicate')` on two 1080x2560 HD1K items with SmallRAFT at 2 iterations equals RAFT's recipe
    per item: InputPadder.pad, the model, unpad, score.  The grid is 135x320, so the level-0 correlation volume holds
    1.87e9 elements, and the metrics take 338 partials per image.  The test peaks at 23 GiB of device memory (measured
    on an H100 80GB).  Counts equal the NumPy oracle's, sums equal it to 1e-12 and the metrics kernel on the recipe's
    prediction bit for bit."""
    import tf_raft_b200 as T
    from tf_raft_b200 import InputPadder, flow_metrics
    _, hd1k = _datasets(tree)
    assert len(hd1k) == 2
    torch.cuda.reset_peak_memory_stats()
    model = T.SmallRAFT(iters=2, iters_pred=2, precision='f16x2', device='cuda:0')
    model.load_params(weights.init_params('small', 7, bias_scale=0.05, norm_jitter=0.1))
    got = T.evaluate(model, hd1k, batch_size=1, per_image=True, protocol='image', padding='replicate', workers=2)
    for k in range(len(hd1k)):
        a, b, f, v = hd1k[k]
        p = InputPadder((1,) + a.shape)
        assert p.padded_size == HD1K and (HD1K[0] // 8 * (HD1K[1] // 8)) ** 2 > 1.8e9
        pa, pb = p.pad(torch.from_numpy(a).cuda()[None], torch.from_numpy(b).cuda()[None])
        pred = p.unpad(model([pa, pb], training=False, last_only=True)[-1]).contiguous()
        c, s = flow_metrics(pred, torch.from_numpy(f).cuda()[None], torch.from_numpy(np.asarray(v, F32)).cuda()[None])
        assert np.array_equal(got['records']['counts'][k], c[0].cpu().numpy())
        assert got['records']['sums'][k].tobytes() == s[0].cpu().numpy().tobytes()
        wc, ws = metrics_np.records(pred.cpu().numpy(), f[None], np.asarray(v, F32)[None])
        np.testing.assert_array_equal(got['records']['counts'][k], wc[0])
        np.testing.assert_allclose(got['records']['sums'][k], ws[0], rtol=1e-12, atol=0)
        assert wc[0, 0] == int((np.asarray(v) != 0).sum()) > 0
    print(f'peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB')
