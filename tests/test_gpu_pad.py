"""GPU: raft_b200_pad_batch bit-exact against np.pad, InputPadder, the loader's replicate padding, the sequence loader,
`evaluate` with RAFT's padding and warm start against hand-written RAFT recipes, and the Sintel / KITTI submission
writers and scripts."""
import collections
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

from oracle import weights
from tf_raft_b200.datasets import frame_utils

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
F32 = np.float32
SIZES = [(1, 1), (5, 7), (13, 3), (436, 1024), (375, 1242), (370, 1224)]


def _np_pad(x, top, bottom, left, right, replicate):
    pads = ((top, bottom), (left, right)) + ((0, 0),) * (x.ndim - 2)
    return np.pad(x, pads, mode='edge') if replicate else np.pad(x, pads, mode='constant')


def _planes(h, w, seed):
    """uint8 frame (h, w, 3), float32 flow (h, w, 2) with NaN, -0.0 and inf in it, float32 valid (h, w)."""
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w, 3)).astype(np.uint8)
    flow = rng.normal(0, 20, (h, w, 2)).astype(F32)
    flow.reshape(-1)[rng.integers(0, flow.size, 3)] = [np.nan, -0.0, np.inf]
    valid = (rng.random((h, w)) < 0.6).astype(F32)
    return img, flow, valid


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _same(t, x):
    """Bit-identical: the same shape, dtype and bytes (NaN payloads and signed zeros included)."""
    got = t.cpu().numpy()
    return got.shape == x.shape and got.dtype == x.dtype and got.tobytes() == x.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['sintel', 'kitti'])
def test_pad_kernel_matches_np_pad(mode):
    """Every plane type in both fills, one launch per size, against np.pad 'edge' / 'constant'.  Destinations start
    filled with a marker, so every pixel must be written."""
    from tf_raft_b200 import _lib
    from tf_raft_b200.preprocess import REPLICATE, ZERO, input_padding, pad_planes
    for k, (h, w) in enumerate(SIZES):
        top, bottom, left, right = input_padding(h, w, mode)
        H, W = h + top + bottom, w + left + right
        srcs = _planes(h, w, k)
        jobs, want = [], []
        for fill in (REPLICATE, ZERO):
            for x in srcs:
                src = _cuda(x)
                dst = torch.full((H, W) + x.shape[2:], 77, dtype=src.dtype, device='cuda')
                jobs.append((src, dst, top, left, fill))
                want.append(_np_pad(x, top, bottom, left, right, fill == REPLICATE))
        _lib.launch_count_reset()
        pad_planes(jobs)
        assert _lib.launch_count() == 1
        for (_, dst, *_), x in zip(jobs, want):
            assert _same(dst, x), (h, w, mode)


def _placed(x, H, W, top, left, replicate):
    """dst(y, x) = src(clamp(y - top), clamp(x - left)) or src(y - top, x - left) inside the source, else 0."""
    h, w = x.shape[:2]
    ys, xs = np.arange(H) - top, np.arange(W) - left
    if replicate:
        return x[np.clip(ys, 0, h - 1)][:, np.clip(xs, 0, w - 1)]
    out = np.zeros((H, W) + x.shape[2:], x.dtype)
    iy, ix = (ys >= 0) & (ys < h), (xs >= 0) & (xs < w)
    out[np.ix_(iy, ix)] = x[np.ix_(ys[iy], xs[ix])]
    return out


@pytest.mark.gpu
def test_pad_kernel_mixed_sizes_and_crops():
    """Items of different source sizes into one padded shape in one launch; targets that crop an axis; and the zero
    fill equal to resize_with_crop_or_pad (the default loader's torch path) bit for bit."""
    from tf_raft_b200 import resize_with_crop_or_pad
    from tf_raft_b200.preprocess import REPLICATE, ZERO, pad_planes, placement
    for mode in ('sintel', 'kitti'):
        jobs, want = [], []
        for k, (h, w) in enumerate([(60, 90), (61, 84), (57, 95), (64, 96), (1, 1)]):
            top, left = placement(h, w, 64, 96, mode)
            for fill in (REPLICATE, ZERO):
                for x in _planes(h, w, 10 + k):
                    src = _cuda(x)
                    jobs.append((src, torch.empty((64, 96) + x.shape[2:], dtype=src.dtype, device='cuda'), top, left,
                                 fill))
                    want.append(np.ascontiguousarray(_np_pad(x, top, 64 - h - top, left, 96 - w - left,
                                                             fill == REPLICATE)))
        pad_planes(jobs)
        for (_, dst, *_), x in zip(jobs, want):
            assert _same(dst, x)
    for (h, w), (H, W) in [((60, 90), (56, 100)), ((60, 90), (64, 88)), ((61, 84), (55, 80)), ((7, 5), (12, 2)),
                           ((436, 1024), (440, 1000)), ((375, 1242), (368, 1248))]:
        for mode in ('sintel', 'kitti'):
            top, left = placement(h, w, H, W, mode)
            jobs, want = [], []
            for fill in (REPLICATE, ZERO):
                for x in _planes(h, w, H + W):
                    src = _cuda(x)
                    jobs.append((src, torch.empty((H, W) + x.shape[2:], dtype=src.dtype, device='cuda'), top, left,
                                 fill))
                    want.append(np.ascontiguousarray(_placed(x, H, W, top, left, fill == REPLICATE)))
            pad_planes(jobs)
            for (src, dst, *_, fill), x in zip(jobs, want):
                assert _same(dst, x), ((h, w), (H, W), mode, fill)
                if fill == ZERO and mode == 'sintel':           # centred: the placement of resize_with_crop_or_pad
                    ref = resize_with_crop_or_pad(src if src.dim() == 3 else src[..., None], H, W)
                    assert _same(dst, ref.cpu().numpy().reshape(tuple(dst.shape)))


@pytest.mark.gpu
def test_input_padder_pads_replicates_and_unpads():
    from tf_raft_b200 import InputPadder, _lib
    from tf_raft_b200.preprocess import input_padding
    rng = np.random.default_rng(3)
    for mode in ('sintel', 'kitti'):
        for h, w in [(61, 84), (436, 1024), (375, 1242), (1, 1)]:
            img = rng.integers(0, 256, (3, h, w, 3)).astype(np.uint8)
            flow = rng.normal(0, 3, (3, h, w, 2)).astype(F32)
            p = InputPadder(img.shape, mode)
            _lib.launch_count_reset()
            a, b = p.pad(_cuda(img), _cuda(flow))
            assert _lib.launch_count() == 1
            top, bottom, left, right = input_padding(h, w, mode)
            pads = ((0, 0), (top, bottom), (left, right), (0, 0))
            assert _same(a, np.pad(img, pads, mode='edge')) and _same(b, np.pad(flow, pads, mode='edge'))
            assert tuple(a.shape[1:3]) == p.padded_size
            assert _same(p.unpad(a), img) and _same(p.unpad(b), flow)
    x = _cuda(rng.integers(0, 256, (2, 64, 96, 3)).astype(np.uint8))
    f = _cuda(rng.normal(0, 1, (2, 64, 96, 2)).astype(F32))
    out = InputPadder(x.shape).pad(x, f)
    assert out[0] is x and out[1] is f                     # aligned: passed through, bit for bit
    with pytest.raises(ValueError):
        InputPadder((1, 60, 90, 3)).pad(x)
    with pytest.raises(TypeError):
        InputPadder(x.shape).pad(x.double())


# --------------------------------------------------------------------------------------------- synthetic datasets
def _write_trees(root, seed=0):
    """Sintel training (flows) and test trees, KITTI training (flow PNGs) and testing trees, of frames whose sizes are
    not multiples of 8 (odd padding in both axes included)."""
    from PIL import Image
    rng = np.random.default_rng(seed)

    def frame(h, w):
        base = rng.integers(0, 256, (h // 6 + 2, w // 6 + 2, 3)).astype(np.uint8)
        return np.kron(base, np.ones((6, 6, 1), np.uint8))[:h, :w]

    def save(path, img):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        Image.fromarray(img).save(path)

    for split, dstypes, scenes in (('training', ('clean',), (('alley_1', 3, 60, 90), ('cave_4', 4, 61, 84))),
                                   ('test', ('clean', 'final'), (('ambush_1', 3, 60, 90), ('bamboo_3', 3, 59, 77)))):
        for scene, n, h, w in scenes:
            for dstype in dstypes:
                for i in range(n):
                    save(os.path.join(root, 'sintel', split, dstype, scene, 'frame_%04d.png' % (i + 1)), frame(h, w))
            if split == 'training':
                d = os.path.join(root, 'sintel', split, 'flow', scene)
                os.makedirs(d, exist_ok=True)
                for i in range(n - 1):
                    frame_utils.write_flow(os.path.join(d, 'frame_%04d.flo' % (i + 1)),
                                           rng.normal(0, 4, (h, w, 2)).astype(F32))
    for split, sizes in (('training', [(60, 90), (61, 84), (60, 90)]), ('testing', [(60, 90), (61, 84), (59, 77)])):
        d = os.path.join(root, 'kitti', split)
        for i, (h, w) in enumerate(sizes):
            for t in (10, 11):
                save(os.path.join(d, 'image_2', '%06d_%d.png' % (i, t)), frame(h, w))
            if split == 'training':
                os.makedirs(os.path.join(d, 'flow_occ'), exist_ok=True)
                frame_utils.write_flow_kitti(os.path.join(d, 'flow_occ', '%06d_10.png' % i),
                                             rng.normal(0, 5, (h, w, 2)).astype(F32), rng.random((h, w)) < 0.7)


@pytest.fixture(scope='module')
def setup(tmp_path_factory):
    import tf_raft_b200 as T
    root = str(tmp_path_factory.mktemp('pad'))
    _write_trees(root)
    model = T.RAFT(iters=2, iters_pred=2, precision='f16x2', device='cuda:0')
    model.load_params(weights.init_params('raft', 1234, bias_scale=0.05, norm_jitter=0.1))
    return root, model


def _dataset(root, name, split=None, dstype='clean'):
    from tf_raft_b200 import datasets as D
    if name == 'sintel':
        return D.MpiSintel(split=split or 'training', root=os.path.join(root, 'sintel'), dstype=dstype)
    return D.KITTI(split=split or 'training', root=os.path.join(root, 'kitti'))


def _padded_frame(x, mode):
    from tf_raft_b200 import InputPadder
    p = InputPadder((1,) + x.shape, mode)
    return p, p.pad(_cuda(x)[None])[0]


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['sintel', 'kitti'])
def test_loader_replicate_batches_equal_input_padder(setup, mode):
    from tf_raft_b200.preprocess import input_padding
    root, _ = setup
    for name in ('sintel', 'kitti'):
        ds = _dataset(root, name)
        for padding in ('replicate', 'zero'):
            k = 0
            for img1, img2, flow, valid, sizes in ds.batches(2, padding=padding, pad_mode=mode, workers=2):
                for j, size in enumerate(sizes):
                    a, b, f, v = ds[k]
                    assert size == a.shape[:2]
                    top, bottom, left, right = input_padding(*size, mode)
                    if padding == 'replicate':
                        assert torch.equal(img1[j:j + 1], _padded_frame(a, mode)[1])
                        assert torch.equal(img2[j:j + 1], _padded_frame(b, mode)[1])
                    else:
                        assert _same(img1[j], _np_pad(a, top, bottom, left, right, False))
                    assert _same(flow[j], _np_pad(f, top, bottom, left, right, False))
                    assert _same(valid[j], _np_pad(np.asarray(v, F32), top, bottom, left, right, False))
                    k += 1
            assert k == len(ds)
    with pytest.raises(ValueError, match='cannot crop'):
        next(_dataset(root, 'sintel').batches(1, target_size=(56, 100), padding='replicate'))


@pytest.mark.gpu
def test_sequences_decode_each_frame_once(setup, monkeypatch):
    import tf_raft_b200.datasets.dataset as dsmod
    from tf_raft_b200.preprocess import input_padding
    root, _ = setup
    ds = _dataset(root, 'sintel')
    calls, lock, read = collections.Counter(), threading.Lock(), dsmod._frame

    def counting(path):
        with lock:
            calls[path] += 1
        return read(path)
    monkeypatch.setattr(dsmod, '_frame', counting)
    scenes = list(ds.sequences(padding='replicate', workers=3, chunk=2))
    paths = {p for pair in ds.image_list for p in pair}
    assert set(calls) == paths and set(calls.values()) == {1}
    monkeypatch.setattr(dsmod, '_frame', read)
    assert [(s[4][0], len(s[4])) for s in scenes] == ds.scenes()
    for frames, flow, valid, size, indices in scenes:
        assert frames.shape[0] == len(indices) + 1 and flow.shape[0] == valid.shape[0] == len(indices)
        top, bottom, left, right = input_padding(*size, 'sintel')
        for t, k in enumerate(indices):
            a, b, f, v = ds[k]
            assert torch.equal(frames[t:t + 1], _padded_frame(a, 'sintel')[1])
            assert torch.equal(frames[t + 1:t + 2], _padded_frame(b, 'sintel')[1])
            assert _same(flow[t], _np_pad(f, top, bottom, left, right, False))
            assert _same(valid[t], _np_pad(np.asarray(v, F32), top, bottom, left, right, False))
    # the zero fill of the sequence loader is the default batches' bytes
    zero = list(ds.sequences(workers=2))
    for (img1, img2, flow, valid, _), k in zip(ds.batches(1, workers=2), range(len(ds))):
        (frames, f, v, _, indices), = [s for s in zero if k in s[4]]
        t = indices.index(k)
        assert torch.equal(img1[0], frames[t]) and torch.equal(img2[0], frames[t + 1])
        assert torch.equal(flow[0].view(torch.int32), f[t].view(torch.int32)) and torch.equal(valid[0], v[t])
    with pytest.raises(ValueError, match='extra_info'):
        next(_dataset(root, 'kitti').sequences())


def _records(pred, flow, valid, max_flow=400):
    from tf_raft_b200 import flow_metrics
    c, s = flow_metrics(pred, _cuda(flow)[None], _cuda(np.asarray(valid, F32))[None], max_flow)
    return c[0].cpu().numpy(), s[0].cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['sintel', 'kitti'])
def test_evaluate_replicate_equals_raft_recipe(setup, mode):
    """Per image: InputPadder.pad, the model, unpad, then the metrics kernel on the original-size ground truth."""
    import tf_raft_b200 as T
    root, model = setup
    for name in ('sintel', 'kitti'):
        ds = _dataset(root, name)
        got = T.evaluate(model, ds, batch_size=2, per_image=True, protocol='image', padding='replicate',
                         pad_mode=mode, workers=2)
        for k in range(len(ds)):
            a, b, f, v = ds[k]
            p, pa = _padded_frame(a, mode)
            pred = model([pa, p.pad(_cuda(b)[None])[0]], training=False, last_only=True)[-1]
            c, s = _records(p.unpad(pred).contiguous(), f, v)
            assert np.array_equal(got['records']['counts'][k], c) and got['records']['sums'][k].tobytes() == s.tobytes()
    # items of different sizes in one padded batch are each scored inside their own rectangle
    ds = _dataset(root, 'kitti')
    one = T.evaluate(model, ds, target_size=(64, 96), per_image=True, padding='replicate', pad_mode=mode)
    three = T.evaluate(model, ds, batch_size=3, target_size=(64, 96), per_image=True, padding='replicate',
                       pad_mode=mode)
    assert np.array_equal(one['records']['counts'], three['records']['counts'])
    assert one['records']['sums'].tobytes() == three['records']['sums'].tobytes()


@pytest.mark.gpu
def test_warm_start_evaluate_equals_predict_video_per_scene(setup):
    import tf_raft_b200 as T
    root, model = setup
    ds = _dataset(root, 'sintel')
    warm = T.evaluate(model, ds, per_image=True, protocol='pixel', padding='replicate', warm_start=True, workers=2)
    cold = T.evaluate(model, ds, per_image=True, protocol='pixel', padding='replicate', workers=2)
    counts, sums = [], []
    for i0, n in ds.scenes():
        items = [ds[k] for k in range(i0, i0 + n)]
        p, first = _padded_frame(items[0][0], 'sintel')
        frames = [first] + [_padded_frame(it[1], 'sintel')[1] for it in items]
        for it, pred in zip(items, model.predict_video(frames, warm_start=True)):
            c, s = _records(p.unpad(pred).contiguous(), it[2], it[3])
            counts.append(c)
            sums.append(s)
        # the warm start resets at each scene: its first pair is the cold record
        assert np.array_equal(warm['records']['counts'][i0], cold['records']['counts'][i0])
        assert warm['records']['sums'][i0].tobytes() == cold['records']['sums'][i0].tobytes()
    assert np.array_equal(warm['records']['counts'], np.array(counts))
    assert warm['records']['sums'].tobytes() == np.array(sums).tobytes()
    assert not np.array_equal(warm['records']['sums'], cold['records']['sums'])     # later pairs were warm-started
    with pytest.raises(ValueError, match='batch_size 1'):
        T.evaluate(model, ds, batch_size=2, warm_start=True)
    with pytest.raises(ValueError, match='extra_info'):
        T.evaluate(model, _dataset(root, 'kitti'), warm_start=True)


@pytest.mark.gpu
def test_sintel_submission(setup, tmp_path):
    import tf_raft_b200 as T
    root, model = setup
    out = str(tmp_path / 'sintel')
    n = T.create_sintel_submission(model, os.path.join(root, 'sintel'), out, workers=2)
    cold_out = str(tmp_path / 'sintel_cold')
    T.create_sintel_submission(model, os.path.join(root, 'sintel'), cold_out, dstypes=('final',), warm_start=False)
    total = 0
    for dstype in ('clean', 'final'):
        ds = _dataset(root, 'sintel', 'test', dstype)
        total += len(ds)
        for s, (i0, npairs) in enumerate(ds.scenes()):
            items = [ds[k] for k in range(i0, i0 + npairs)]
            p, first = _padded_frame(items[0][0], 'sintel')
            frames = [first] + [_padded_frame(it[1], 'sintel')[1] for it in items]
            warm = list(model.predict_video(frames, warm_start=True))
            pairs = [model([frames[t], frames[t + 1]], training=False, last_only=True)[-1] for t in range(npairs)]
            assert torch.equal(warm[0], pairs[0])                 # every scene, the second included, starts cold
            for t, k in enumerate(range(i0, i0 + npairs)):
                scene, index = ds.extra_info[k]
                got = frame_utils.read_flow(os.path.join(out, dstype, scene, 'frame%04d.flo' % (index + 1)))
                assert got.shape == items[t][0].shape[:2] + (2,)
                assert got.tobytes() == p.unpad(warm[t])[0].cpu().numpy().tobytes()
                if dstype == 'final':
                    cold = frame_utils.read_flow(os.path.join(cold_out, dstype, scene, 'frame%04d.flo' % (index + 1)))
                    assert cold.tobytes() == p.unpad(pairs[t])[0].cpu().numpy().tobytes()
    assert n == total
    assert sum(len(f) for _, _, f in os.walk(out)) == total


@pytest.mark.gpu
def test_kitti_submission(setup, tmp_path):
    import tf_raft_b200 as T
    from tf_raft_b200.datasets import read_flow_kitti_batch
    from tf_raft_b200.submission import kitti_flow_for_png
    root, model = setup
    out = str(tmp_path / 'kitti')
    assert T.create_kitti_submission(model, os.path.join(root, 'kitti'), out, batch_size=2, workers=2) == 3
    ds = _dataset(root, 'kitti', 'testing')
    assert sorted(os.listdir(out)) == sorted(e[0] for e in ds.extra_info)
    for k in range(len(ds)):
        a, b, (frame_id,) = ds[k]
        p, pa = _padded_frame(a, 'kitti')
        pred = p.unpad(model([pa, p.pad(_cuda(b)[None])[0]], training=False, last_only=True)[-1])[0]
        clamped = kitti_flow_for_png(pred).cpu().numpy()
        want = ((64.0 * clamped + 2 ** 15).astype(np.uint16).astype(F32) - 2 ** 15) / 64.0
        flow, valid = read_flow_kitti_batch([os.path.join(out, frame_id)])
        assert flow.shape == (1,) + a.shape[:2] + (2,)
        assert _same(flow[0], want.astype(F32)) and bool((valid == 1).all())


def _script(*args):
    proc = subprocess.run([sys.executable, os.path.join(ROOT, 'scripts', args[0])] + list(args[1:]),
                          capture_output=True, text=True, timeout=900)
    assert proc.returncode == 0, proc.stdout[-3000:] + proc.stderr[-3000:]
    return json.loads(proc.stdout.strip().splitlines()[-1])


@pytest.mark.gpu
def test_submit_and_evaluate_scripts(setup, tmp_path):
    root, model = setup
    ck = str(tmp_path / 'ck' / 'model')
    model.save_weights(ck)
    out = _script('submit.py', 'sintel', '--root', os.path.join(root, 'sintel'), '--checkpoint', ck, '--out',
                  str(tmp_path / 'sub'), '--iters', '2', '--workers', '2')
    assert out['files'] == 2 * len(_dataset(root, 'sintel', 'test')) and out['warm_start']
    for dstype in ('clean', 'final'):
        for scene in ('ambush_1', 'bamboo_3'):
            assert sorted(os.listdir(tmp_path / 'sub' / dstype / scene)) == ['frame0001.flo', 'frame0002.flo']
    out = _script('submit.py', 'kitti', '--root', os.path.join(root, 'kitti'), '--checkpoint', ck, '--out',
                  str(tmp_path / 'kitti'))
    assert out['files'] == 3 and out['iters'] == 24 and len(os.listdir(tmp_path / 'kitti')) == 3
    res = _script('evaluate.py', 'sintel', '--root', os.path.join(root, 'sintel'), '--checkpoint', ck, '--iters', '2',
                  '--padding', 'replicate', '--warm-start', '--workers', '2')
    assert res['pixels'] == 2 * 60 * 90 + 3 * 61 * 84                  # every pixel of the five original frames
    assert res['padding'] == 'replicate' and res['warm_start'] and res['pairs'] == 5
