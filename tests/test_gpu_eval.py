"""GPU: the KITTI flow-PNG decoder against the NumPy reader, the metrics kernel against oracle/metrics_np.py, the
'keras' aggregation against the existing metric, `evaluate` end to end and the training loader against
`augmentor.batch`."""
import os
import random
import struct
import zlib

import numpy as np
import pytest
import torch

from oracle import metrics_np, weights
from tf_raft_b200.datasets import frame_utils

F32 = np.float32


# --------------------------------------------------------------------------------------------- a PNG encoder
def _filter_row(cur, prev, ft):
    """PNG filter type ft of one row of bytes (int32 arrays), bpp 6, from the unfiltered row and the one above."""
    a = np.concatenate([np.zeros(6, np.int32), cur[:-6]])
    c = np.concatenate([np.zeros(6, np.int32), prev[:-6]])
    b = prev
    if ft == 0:
        pred = np.zeros_like(cur)
    elif ft == 1:
        pred = a
    elif ft == 2:
        pred = b
    elif ft == 3:
        pred = (a + b) >> 1
    else:
        pa, pb, pc = np.abs(b - c), np.abs(a - c), np.abs(a + b - 2 * c)
        pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    return ((cur - pred) & 255).astype(np.uint8)


def encode_png16(path, rgb16, filters, n_idat=3):
    """16-bit RGB PNG of an (H, W, 3) uint16 array with row y filtered by filters[y % len(filters)], its zlib stream
    split over n_idat IDAT chunks."""
    h, w, _ = rgb16.shape
    rows = rgb16.astype('>u2').view(np.uint8).reshape(h, 6 * w).astype(np.int32)
    prev = np.zeros(6 * w, np.int32)
    out = []
    for y in range(h):
        ft = filters[y % len(filters)]
        out.append(bytes([ft]) + _filter_row(rows[y], prev, ft).tobytes())
        prev = rows[y]
    z = zlib.compress(b''.join(out))
    cut = [len(z) * k // n_idat for k in range(n_idat + 1)]

    def chunk(kind, body):
        return struct.pack('>I', len(body)) + kind + body + struct.pack('>I', zlib.crc32(kind + body) & 0xffffffff)
    with open(path, 'wb') as f:
        f.write(b'\x89PNG\r\n\x1a\n' + chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, 16, 2, 0, 0, 0)) +
                b''.join(chunk(b'IDAT', z[cut[k]:cut[k + 1]]) for k in range(n_idat)) + chunk(b'IEND', b''))


def _rgb16(h, w, seed):
    rng = np.random.default_rng(seed)
    rgb = rng.integers(0, 65536, (h, w, 3)).astype(np.uint16)
    rgb[..., 2] = rng.integers(0, 2, (h, w))
    return rgb


def _expected(rgb):
    f = rgb.astype(F32)
    return ((f[..., :2] - 2 ** 15) / 64.0).astype(F32), f[..., 2]


def _decode_files(paths):
    from tf_raft_b200.datasets.png16 import decode_png16, pack_rows
    inflated = [frame_utils.inflate_png16(p) for p in paths]
    offsets, total = pack_rows(inflated)
    data = torch.from_numpy(np.frombuffer(b''.join(r for r, _, _ in inflated), np.uint8).copy()).cuda()
    assert data.numel() == total
    out = decode_png16(data, [(o, h, w) for o, (_, h, w) in zip(offsets, inflated)], paths)
    return [(f.cpu().numpy(), v.cpu().numpy()) for f, v in out]


FILTERS = {'none': [0], 'sub': [1], 'up': [2], 'average': [3], 'paeth': [4], 'mixed': [0, 1, 2, 3, 4, 4, 3, 1, 2]}
SMALL = [(1, 1), (1, 13), (5, 7), (3, 2), (9, 31)]


@pytest.mark.gpu
def test_png_decoder_small_sizes_against_the_numpy_reader(tmp_path):
    """Every filter forced on every row, and all five mixed, at small sizes decoded in one mixed-size launch: equal to
    read_flow_kitti (the NumPy reader) bit for bit."""
    paths = []
    for (h, w) in SMALL:
        for name, filters in FILTERS.items():
            p = str(tmp_path / f'{name}_{h}x{w}.png')
            encode_png16(p, _rgb16(h, w, h * 100 + w + len(paths)), filters, n_idat=1 + len(paths) % 3)
            paths.append(p)
    for p, (flow, valid) in zip(paths, _decode_files(paths)):
        want_flow, want_valid = frame_utils.read_flow_kitti(p)
        assert flow.dtype == want_flow.dtype and flow.shape == want_flow.shape
        np.testing.assert_array_equal(flow, want_flow, err_msg=p)
        np.testing.assert_array_equal(valid, want_valid, err_msg=p)


@pytest.mark.gpu
def test_png_decoder_kitti_sizes(tmp_path):
    """375x1242 and 376x1241 with each filter on every row, in one batch with a small file.  The mixed file of each
    size is compared with the NumPy reader, the rest with the encoded values (which that reader returns, above)."""
    paths, want = [], []
    for (h, w) in [(375, 1242), (376, 1241)]:
        for k, (name, filters) in enumerate(FILTERS.items()):
            rgb = _rgb16(h, w, 7 * k + h)
            p = str(tmp_path / f'{name}_{h}x{w}.png')
            encode_png16(p, rgb, filters)
            paths.append(p)
            want.append(frame_utils.read_flow_kitti(p) if name == 'mixed' else _expected(rgb))
    p = str(tmp_path / 'small.png')
    encode_png16(p, _rgb16(2, 3, 1), [4])
    paths.append(p)
    want.append(frame_utils.read_flow_kitti(p))
    for p, got, w in zip(paths, _decode_files(paths), want):
        np.testing.assert_array_equal(got[0], w[0], err_msg=p)
        np.testing.assert_array_equal(got[1], w[1], err_msg=p)


@pytest.mark.gpu
def test_read_flow_kitti_batch_on_written_files(tmp_path):
    """Files from write_flow_kitti and, where it imports, cv2.imwrite (libpng picks the filters) -- equal sizes."""
    from tf_raft_b200.datasets import read_flow_kitti_batch
    rng = np.random.default_rng(3)
    paths = []
    for i in range(3):
        p = str(tmp_path / f'w{i}.png')
        frame_utils.write_flow_kitti(p, rng.normal(0, 30, (375, 1242, 2)).astype(F32),
                                     (rng.random((375, 1242)) < 0.5).astype(F32))
        paths.append(p)
    try:
        import cv2
        for i in range(2):
            p = str(tmp_path / f'cv{i}.png')
            rgb = np.clip(64 * rng.normal(0, 30, (375, 1242, 3)) + 2 ** 15, 0, 65535).astype(np.uint16)
            rgb[..., 2] = rng.integers(0, 2, (375, 1242))
            assert cv2.imwrite(p, rgb[..., ::-1])
            paths.append(p)
    except ImportError:
        pass
    flow, valid = read_flow_kitti_batch(paths)
    assert flow.shape == (len(paths), 375, 1242, 2) and valid.shape == (len(paths), 375, 1242)
    for i, p in enumerate(paths):
        wf, wv = frame_utils.read_flow_kitti(p)
        np.testing.assert_array_equal(flow[i].cpu().numpy(), wf, err_msg=p)
        np.testing.assert_array_equal(valid[i].cpu().numpy(), wv, err_msg=p)
    with pytest.raises(ValueError, match='equal sizes'):
        small = str(tmp_path / 'small.png')
        frame_utils.write_flow_kitti(small, np.zeros((4, 5, 2), F32))
        read_flow_kitti_batch([paths[0], small])


@pytest.mark.gpu
def test_png_decoder_rejects_malformed_streams(tmp_path):
    """A truncated file raises on the host naming it; a bad filter byte the host never saw is reported by the kernel's
    status word, naming the file, and the device stays usable."""
    from tf_raft_b200.datasets import read_flow_kitti_batch
    from tf_raft_b200.datasets.png16 import decode_png16
    good = str(tmp_path / 'good.png')
    encode_png16(good, _rgb16(6, 9, 2), [4, 1])
    raw = open(good, 'rb').read()
    cut = str(tmp_path / 'truncated.png')
    open(cut, 'wb').write(raw[:len(raw) // 2])
    with pytest.raises(ValueError, match='truncated.png'):
        read_flow_kitti_batch([good, cut])
    rows, h, w = frame_utils.inflate_png16(good)
    bad = bytearray(rows)
    bad[3 * (1 + 6 * w)] = 9                                      # row 3's filter byte
    data = torch.from_numpy(np.frombuffer(rows + bytes(bad), np.uint8).copy()).cuda()
    with pytest.raises(ValueError, match=r'second\.png: unknown PNG filter type in row 3'):
        decode_png16(data, [(0, h, w), (len(rows), h, w)], ['first.png', 'second.png'])
    flow, valid = read_flow_kitti_batch([good])
    np.testing.assert_array_equal(flow[0].cpu().numpy(), frame_utils.read_flow_kitti(good)[0])


# --------------------------------------------------------------------------------------------- metrics kernel
def _records(pred, gt, valid, max_flow=400):
    from tf_raft_b200 import flow_metrics
    c, s = flow_metrics(torch.from_numpy(pred).cuda(), torch.from_numpy(gt).cuda(),
                        None if valid is None else torch.from_numpy(valid).cuda(), max_flow)
    return c.cpu().numpy(), s.cpu().numpy()


def _check(pred, gt, valid, max_flow=400):
    c, s = _records(pred, gt, valid, max_flow)
    wc, ws = metrics_np.records(pred, gt, valid, max_flow)
    np.testing.assert_array_equal(c, wc)
    fin = np.isfinite(ws)
    np.testing.assert_array_equal(s[~fin], ws[~fin])
    np.testing.assert_allclose(s[fin], ws[fin], rtol=1e-12, atol=0)
    return c, s


def _random_case(B, H, W, seed):
    rng = np.random.default_rng(seed)
    gt = rng.normal(0, 60, (B, H, W, 2)).astype(F32)
    pred = (gt + rng.normal(0, 3, gt.shape)).astype(F32)
    valid = (rng.random((B, H, W)) < 0.8).astype(F32)
    return pred, gt, valid


@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(1, 1, 1), (3, 7, 13), (2, 64, 96), (4, 436, 1024), (8, 1088, 1920)])
def test_metrics_kernel_against_numpy(shape):
    pred, gt, valid = _random_case(*shape, seed=sum(shape))
    _check(pred, gt, valid)
    _check(pred, gt, None, max_flow=None)
    _check(pred, gt, valid, max_flow=50)


@pytest.mark.gpu
def test_metrics_kernel_edge_cases():
    top = np.float32(400)
    below = np.nextafter(top, F32(0))
    rows = [  # (gt, pred, valid)
        ((3, 4), (3, 4), 1), ((top, 0), (top, 0), 1), ((below, 0), (below, 0), 1), ((0, top), (1, top), 1),
        ((10, 0), (11, 0), 1), ((10, 0), (13, 0), 1), ((10, 0), (15, 0), 1), ((0, 10), (0, 7), 1), ((0, 0), (0, 5), 1),
        ((0, 0), (0, 3), 1), ((80, 0), (84, 0), 1), ((80, 0), (84.01, 0), 1), ((np.nan, 0), (0, 0), 1),
        ((0, 0), (np.nan, 0), 1), ((0, 0), (np.inf, 0), 1), ((np.inf, 0), (np.inf, 0), 1), ((-np.inf, 1), (0, 0), 1),
        ((1, 1), (2, 2), np.nan), ((1, 1), (2, 2), 0), ((1, 1), (9, 9), -0.5), ((2, 0), (2, 1), 1),
    ]
    gt = np.array([r[0] for r in rows], F32).reshape(1, 1, -1, 2)
    pred = np.array([r[1] for r in rows], F32).reshape(1, 1, -1, 2)
    valid = np.array([r[2] for r in rows], F32).reshape(1, 1, -1)
    assert F32(4) / F32(80) == F32(0.05)                          # epe / mag exactly float32(0.05): not an outlier
    for mf in (400, None):
        c, _ = _check(pred, gt, valid, mf)
        c2, _ = _check(np.concatenate([pred] * 3), np.concatenate([gt] * 3), np.concatenate([valid, np.zeros_like(valid), valid]),
                       mf)
        assert (c2[1] == 0).all() and (c2[0] == c[0]).all()      # an all-invalid image, between two others
    c, s = _records(pred, gt, valid, 400)
    assert np.isnan(s[0])                                         # NaN epe enters the sum


@pytest.mark.gpu
def test_metrics_records_do_not_depend_on_batch_or_run():
    pred, gt, valid = _random_case(8, 436, 1024, seed=11)
    c8, s8 = _records(pred, gt, valid)
    again = _records(pred, gt, valid)
    np.testing.assert_array_equal(c8, again[0])
    assert s8.tobytes() == again[1].tobytes()
    for b in (0, 5):
        c1, s1 = _records(pred[b:b + 1], gt[b:b + 1], valid[b:b + 1])
        np.testing.assert_array_equal(c1[0], c8[b])
        assert s1[0].tobytes() == s8[b].tobytes()


@pytest.mark.gpu
def test_keras_aggregation_matches_end_point_error():
    from tf_raft_b200 import EndPointError, FlowMetrics, end_point_error
    m, ref = FlowMetrics(), EndPointError()
    for k in range(4):
        pred, gt, valid = _random_case(3, 40, 56, seed=30 + k)
        pred, gt, valid = (torch.from_numpy(a).cuda() for a in (pred, gt, valid))
        m.update_state(gt, pred, valid)
        ref.update_state([gt, valid], [pred])
        one = end_point_error([gt, valid], pred)
        single = FlowMetrics()
        single.update_state(gt, pred, valid)
        got = single.result()
        for key in ('epe', 'u1', 'u3', 'u5'):
            assert got[key] == pytest.approx(float(one[key]), rel=1e-6)
    got, want = m.result(), ref.result()
    for key in ('epe', 'u1', 'u3', 'u5'):
        assert got[key] == pytest.approx(want[key], rel=1e-6)


# --------------------------------------------------------------------------------------------- end to end
def _write_eval_trees(root, seed=0):
    """A Sintel-layout tree of 60x90 frames and a KITTI-layout tree with 60x90 and 61x84 pairs."""
    from PIL import Image
    rng = np.random.default_rng(seed)

    def frame(h, w):
        base = rng.integers(0, 256, (h // 6 + 2, w // 6 + 2, 3)).astype(np.uint8)
        return np.kron(base, np.ones((6, 6, 1), np.uint8))[:h, :w]

    for scene, n in (('alley_1', 3), ('cave_4', 2)):
        d = os.path.join(root, 'sintel', 'training', 'clean', scene)
        os.makedirs(d, exist_ok=True)
        os.makedirs(os.path.join(root, 'sintel', 'training', 'flow', scene), exist_ok=True)
        for i in range(n):
            Image.fromarray(frame(60, 90)).save(os.path.join(d, 'frame_%04d.png' % (i + 1)))
        for i in range(n - 1):
            frame_utils.write_flow(os.path.join(root, 'sintel', 'training', 'flow', scene, 'frame_%04d.flo' % (i + 1)),
                                   rng.normal(0, 4, (60, 90, 2)).astype(F32))
    d = os.path.join(root, 'kitti', 'training')
    os.makedirs(os.path.join(d, 'image_2'), exist_ok=True)
    os.makedirs(os.path.join(d, 'flow_occ'), exist_ok=True)
    for i, (h, w) in enumerate([(60, 90), (61, 84), (60, 90), (60, 90), (61, 84)]):
        for t in (10, 11):
            Image.fromarray(frame(h, w)).save(os.path.join(d, 'image_2', '%06d_%d.png' % (i, t)))
        rgb = np.empty((h, w, 3), np.uint16)
        rgb[..., :2] = np.clip(64 * rng.normal(0, 5, (h, w, 2)) + 2 ** 15, 0, 65535)
        rgb[..., 2] = rng.random((h, w)) < 0.7
        encode_png16(os.path.join(d, 'flow_occ', '%06d_10.png' % i), rgb, [1, 4, 2, 3, 0])


@pytest.fixture(scope='module')
def eval_setup(tmp_path_factory):
    import tf_raft_b200 as T
    root = str(tmp_path_factory.mktemp('eval'))
    _write_eval_trees(root)
    model = T.RAFT(iters=2, iters_pred=2, precision='f16x2', device='cuda:0')
    model.load_params(weights.init_params('raft', 1234, bias_scale=0.05, norm_jitter=0.1))
    return root, model


def _scored_one_by_one(model, ds, max_flow):
    """Each item padded alone, the prediction cropped back and scored by the NumPy restatement."""
    from tf_raft_b200 import pad_to_multiple, resize_with_crop_or_pad
    counts, sums = [], []
    for i in range(len(ds)):
        img1, img2, flow, valid = ds[i]
        a, (h, w) = pad_to_multiple(torch.from_numpy(img1).cuda())
        b, _ = pad_to_multiple(torch.from_numpy(img2).cuda())
        pred = model([a[None], b[None]], training=False, last_only=True)[-1]
        pred = resize_with_crop_or_pad(pred, h, w).cpu().numpy()
        c, s = metrics_np.records(pred, flow[None], np.asarray(valid, F32)[None], max_flow)
        counts.append(c[0])
        sums.append(s[0])
    return np.array(counts), np.array(sums)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['sintel', 'kitti'])
def test_evaluate_end_to_end(eval_setup, name):
    import tf_raft_b200 as T
    from tf_raft_b200 import datasets as D
    root, model = eval_setup
    ds = D.MpiSintel(root=os.path.join(root, 'sintel')) if name == 'sintel' else D.KITTI(root=os.path.join(root, 'kitti'))
    want_c, want_s = _scored_one_by_one(model, ds, 400)
    r1 = T.evaluate(model, ds, batch_size=1, per_image=True, protocol='image', workers=2)
    r3 = T.evaluate(model, ds, batch_size=3, per_image=True, protocol='image', workers=3)
    for r in (r1, r3):
        np.testing.assert_array_equal(r['records']['counts'], want_c)
        np.testing.assert_allclose(r['records']['sums'], want_s, rtol=1e-12)
    np.testing.assert_array_equal(r1['records']['counts'], r3['records']['counts'])
    assert r1['records']['sums'].tobytes() == r3['records']['sums'].tobytes()
    # 'keras' is a loop of test_step over the loader's batches
    keras = T.evaluate(model, ds, batch_size=2, protocol='keras')
    model.compile()
    for image1, image2, flow, valid, sizes in ds.batches(2):
        res = model.test_step((image1, image2, flow, valid))
    for key in ('epe', 'u1', 'u3', 'u5'):
        assert keras[key] == pytest.approx(res[key], rel=1e-6)
    pixel = T.evaluate(model, ds, protocol='pixel')
    assert pixel['epe'] == pytest.approx(want_s.sum() / want_c[:, 0].sum(), rel=1e-12)
    assert pixel['pixels'] == want_c[:, 0].sum()


@pytest.mark.gpu
def test_eval_loader_groups_by_padded_shape(eval_setup):
    from tf_raft_b200 import datasets as D
    root, _ = eval_setup
    ds = D.KITTI(root=os.path.join(root, 'kitti'))
    shapes = [(tuple(b[0].shape), b[4]) for b in ds.batches(4)]
    assert shapes == [((1, 64, 96, 3), [(60, 90)]), ((1, 64, 88, 3), [(61, 84)]),
                      ((2, 64, 96, 3), [(60, 90), (60, 90)]), ((1, 64, 88, 3), [(61, 84)])]
    img1, _, flow, valid, _ = next(iter(ds.batches(1, target_size=(56, 100))))
    item = ds[0]
    assert img1.shape == (1, 56, 100, 3) and img1.dtype == torch.uint8
    np.testing.assert_array_equal(img1[0, :, 5:95].cpu().numpy(), item[0][2:58])
    np.testing.assert_array_equal(flow[0, :, 5:95].cpu().numpy(), item[2][2:58])
    assert float(valid[0, :, :5].abs().sum()) == 0 and float(flow[0, :, 95:].abs().sum()) == 0


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['sintel', 'kitti'])
def test_training_loader_matches_augmentor_batch(eval_setup, name):
    from tf_raft_b200 import datasets as D
    root, _ = eval_setup
    aug = {'crop_size': (40, 64), 'min_scale': -0.2, 'max_scale': 0.4, 'do_flip': True}
    ds = D.MpiSintel(aug, root=os.path.join(root, 'sintel')) if name == 'sintel' else \
        D.KITTI(aug, root=os.path.join(root, 'kitti'))
    plain = D.MpiSintel(root=os.path.join(root, 'sintel')) if name == 'sintel' else \
        D.KITTI(root=os.path.join(root, 'kitti'))
    np.random.seed(5)
    random.seed(5)
    got = [tuple(t.cpu() for t in b) for b in ds.batches(2, workers=3)]
    np.random.seed(5)
    random.seed(5)
    items = [plain[i] for i in range(len(plain))]
    want = []
    for k in range(0, len(items), 2):
        samples = [it if ds.sparse else it[:3] for it in items[k:k + 2]]
        want.append(tuple(t.cpu() for t in ds.augmentor.batch(samples)))
    assert len(got) == len(want) == -(-len(items) // 2)
    for g, w in zip(got, want):
        for a, b in zip(g, w):
            assert torch.equal(a, b)
