"""The dataset classes against the reference's own file lists and items (tests/golden/datasets.npz, written by
tests/golden/make_datasets_golden.py from the reference's dataset.py on the tree `make_tree` builds), the readers, and
the metric aggregations.  No GPU needed."""
import os
import struct

import numpy as np
import pytest

from tf_raft_b200.datasets import frame_utils

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'datasets.npz')

SINTEL_SCENES = {'alley_1': (4, 'RGB'), 'bamboo_2': (3, 'L'), 'cave_4': (3, 'RGBA'), 'market_5': (2, 'RGB')}


def write_pfm(path, data, little_endian):
    """PFM writer: 'PF' for (H, W, 3), 'Pf' for (H, W); rows bottom-up; a negative scale marks little endian."""
    data = np.asarray(data, np.float32)
    with open(path, 'wb') as f:
        f.write(b'PF\n' if data.ndim == 3 else b'Pf\n')
        f.write(b'%d %d\n' % (data.shape[1], data.shape[0]))
        f.write(b'-1.0\n' if little_endian else b'1.0\n')
        f.write(np.ascontiguousarray(np.flipud(data)).astype('<f4' if little_endian else '>f4').tobytes())


def make_tree(root, seed=0):
    """Synthetic Sintel, FlyingChairs, FlyingThings3D, KITTI and HD1K layouts under `root`, all content from `seed`."""
    from PIL import Image
    rng = np.random.default_rng(seed)

    def mk(path):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        return path

    def img(path, h, w, mode='RGB'):
        shape = (h, w) if mode == 'L' else (h, w, len(mode))
        Image.fromarray(rng.integers(0, 256, shape, dtype=np.uint8), mode).save(mk(path))

    def flo(path, h, w, edge=False):
        f = rng.normal(0, 5, (h, w, 2)).astype(np.float32)
        if edge:                              # the dense valid's boundary: |u| = 1000 is invalid, just below is valid
            f[0, 0, 0], f[0, 1, 1], f[1, 0, 0], f[1, 1, 1] = 1000, -1000, np.nextafter(np.float32(1000), 0), -999
        frame_utils.write_flow(mk(path), f)

    def kitti_flow(path, h, w):
        f = rng.normal(0, 20, (h, w, 2)).astype(np.float32)
        valid = (rng.random((h, w)) < 0.6).astype(np.float32)
        frame_utils.write_flow_kitti(mk(path), f, valid)

    j = os.path.join
    h, w = 6, 10
    for split in ('training', 'test'):
        for dstype in ('clean', 'final'):
            for scene, (n, mode) in SINTEL_SCENES.items():
                for i in range(n):
                    img(j(root, 'sintel', split, dstype, scene, 'frame_%04d.png' % (i + 1)), h, w, mode)
    for scene, (n, _) in SINTEL_SCENES.items():
        for i in range(n - 1):
            flo(j(root, 'sintel', 'training', 'flow', scene, 'frame_%04d.flo' % (i + 1)), h, w, edge=scene == 'alley_1')
    for i in range(5):
        img(j(root, 'chairs', 'data', '%05d_img1.ppm' % (i + 1)), 5, 7)
        img(j(root, 'chairs', 'data', '%05d_img2.ppm' % (i + 1)), 5, 7)
        flo(j(root, 'chairs', 'data', '%05d_flow.flo' % (i + 1)), 5, 7)
    np.savetxt(j(root, 'chairs', 'split.txt'), [1, 2, 1, 1, 2], fmt='%d')
    k = 0
    for letter in ('A', 'B'):
        for seq in ('0000', '0001'):
            for cam in ('left', 'right'):
                for t in range(6, 9 + (seq == '0001')):
                    img(j(root, 'things', 'frames_cleanpass', 'TRAIN', letter, seq, cam, '%04d.png' % t), 4, 6)
                    for d, tag in (('into_future', 'IntoFuture'), ('into_past', 'IntoPast')):
                        name = 'OpticalFlow%s_%04d_%s.pfm' % (tag, t, cam[0].upper())
                        write_pfm(mk(j(root, 'things', 'optical_flow', 'TRAIN', letter, seq, d, cam, name)),
                                  rng.normal(0, 3, (4, 6, 3)), little_endian=k % 2 == 0)
                        k += 1
    for split, n in (('training', 3), ('testing', 2)):
        for i in range(n):
            hh, ww = (6, 10) if i % 2 == 0 else (7, 9)
            img(j(root, 'kitti', split, 'image_2', '%06d_10.png' % i), hh, ww)
            img(j(root, 'kitti', split, 'image_2', '%06d_11.png' % i), hh, ww)
            if split == 'training':
                kitti_flow(j(root, 'kitti', split, 'flow_occ', '%06d_10.png' % i), hh, ww)
    for seq, n in enumerate((3, 2, 4)):
        for t in range(n):
            img(j(root, 'hd1k', 'hd1k_input', 'image_2', '%06d_%04d.png' % (seq, t)), 5, 8)
            kitti_flow(j(root, 'hd1k', 'hd1k_flow_gt', 'flow_occ', '%06d_%04d.png' % (seq, t)), 5, 8)


def configs(D, root):
    """The datasets the golden file records, built with module D (the reference's dataset.py or ours)."""
    j = os.path.join
    sintel = D.MpiSintel(root=j(root, 'sintel'))
    chairs_train = D.FlyingChairs(split_txt=j(root, 'chairs', 'split.txt'), root=j(root, 'chairs', 'data'))
    things = D.FlyingThings3D(root=j(root, 'things'))
    kitti = D.KITTI(root=j(root, 'kitti'))
    hd1k = D.HD1K(root=j(root, 'hd1k'))
    out = {
        'sintel_clean': sintel,
        'sintel_final': D.MpiSintel(root=j(root, 'sintel'), dstype='final'),
        'sintel_test': D.MpiSintel(root=j(root, 'sintel'), split='test'),
        'chairs_train': chairs_train,
        'chairs_val': D.FlyingChairs(split='validation', split_txt=j(root, 'chairs', 'split.txt'),
                                     root=j(root, 'chairs', 'data')),
        'things_clean': things,
        'kitti_train': kitti,
        'kitti_test': D.KITTI(split='testing', root=j(root, 'kitti')),
        'hd1k': hd1k,
        'combo': 2 * kitti + hd1k,
    }
    shuffled = 2 * things + chairs_train
    np.random.seed(7)
    shuffled.shuffle()
    out['shuffled'] = shuffled
    return out


# (dataset, key): Sintel items are found by (scene, frame) since scene order follows os.listdir.
ITEMS = [('sintel_clean', ('bamboo_2', 0)), ('sintel_clean', ('cave_4', 1)), ('sintel_clean', ('alley_1', 0)),
         ('sintel_test', ('alley_1', 1)), ('kitti_train', 0), ('kitti_train', 1), ('kitti_test', 1),
         ('things_clean', 0), ('things_clean', -1), ('chairs_train', 1), ('chairs_val', 0), ('hd1k', 3)]


def item_index(ds, key):
    if isinstance(key, tuple):
        return [tuple(e) for e in ds.extra_info].index(key)
    return key % len(ds)


def item_tag(name, key):
    return f'{name}/{key[0]}_{key[1]}' if isinstance(key, tuple) else f'{name}/{key}'


def describe(ds, root):
    rel = lambda p: os.path.relpath(p, root)  # noqa: E731
    return {'images': np.array([[rel(a), rel(b)] for a, b in ds.image_list], dtype=str).reshape(-1, 2),
            'flows': np.array([rel(p) for p in ds.flow_list], dtype=str),
            'extra': np.array(['/'.join(str(x) for x in e) for e in ds.extra_info], dtype=str),
            'flags': np.array([bool(ds.is_test), bool(ds.sparse)])}


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('datasets'))
    make_tree(root)
    from tf_raft_b200 import datasets as D
    return root, configs(D, root)


@pytest.fixture(scope='module')
def ds_golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize('name', ['sintel_final', 'sintel_test', 'chairs_train', 'chairs_val', 'things_clean',
                                  'kitti_train', 'kitti_test', 'hd1k', 'combo', 'shuffled', 'sintel_clean'])
def test_file_lists_match_the_reference(tree, ds_golden, name):
    root, ds = tree
    got = describe(ds[name], root)
    for field in ('images', 'flows', 'extra', 'flags'):
        want = ds_golden[f'{name}/{field}']
        if name.startswith('sintel') and field != 'flags':
            # os.listdir order depends on the filesystem: compare per scene, and that scenes come in listdir order
            for s in SINTEL_SCENES:
                np.testing.assert_array_equal(_scene_rows(got[field], field, s), _scene_rows(want, field, s),
                                              err_msg=f'{name} {field} {s}')
        else:
            np.testing.assert_array_equal(got[field], want, err_msg=f'{name} {field}')
    if name.startswith('sintel'):
        order = list(dict.fromkeys(str(e).split('/')[0] for e in got['extra']))
        listdir = os.listdir(os.path.dirname(os.path.join(root, got['images'][0][0])) + '/..')
        assert order == [s for s in listdir if s in order]


def _scene_rows(rows, field, scene):
    """Rows of a Sintel list that belong to `scene` (extra_info 'scene/i'; paths sintel/<split>/<dir>/<scene>/...)."""
    pick = (lambda r: str(r).split('/')[0]) if field == 'extra' else \
        (lambda r: str(r[0] if field == 'images' else r).split('/')[3])
    return np.array([r for r in rows if pick(r) == scene], dtype=str)


def test_items_match_the_reference(tree, ds_golden):
    root, ds = tree
    for name, key in ITEMS:
        got = ds[name][item_index(ds[name], key)]
        tag = item_tag(name, key)
        if ds[name].is_test:
            assert len(got) == 3
            assert '/'.join(str(x) for x in got[2]) == str(ds_golden[f'item/{tag}/2'])
            got = got[:2]
        for k, a in enumerate(got):
            want = ds_golden[f'item/{tag}/{k}']
            assert a.dtype == want.dtype and a.shape == want.shape, (tag, k, a.dtype, want.dtype, a.shape, want.shape)
            np.testing.assert_array_equal(a, want, err_msg=f'{tag} [{k}]')


def test_item_edge_cases(tree):
    """The grayscale scene is tiled to 3 channels, RGBA is cut to RGB, |u| = 1000 is invalid, KITTI's valid is float."""
    root, ds = tree
    s = ds['sintel_clean']
    g = s[item_index(s, ('bamboo_2', 0))]
    assert g[0].shape == (6, 10, 3) and np.array_equal(g[0][..., 0], g[0][..., 2])
    assert s[item_index(s, ('cave_4', 0))][0].shape == (6, 10, 3)
    valid = s[item_index(s, ('alley_1', 0))][3]
    assert valid.dtype == bool and not valid[0, 0] and not valid[0, 1] and valid[1, 0] and valid[1, 1]
    k = ds['kitti_train'][0]
    assert k[2].dtype == np.float32 and k[3].dtype == np.float32 and set(np.unique(k[3])) <= {0.0, 1.0}


def test_container_quirks(tree):
    root, ds = tree
    sintel, kitti = ds['sintel_clean'], ds['kitti_train']
    both = sintel + kitti
    assert not both.sparse and both.extra_info == sintel.extra_info          # the left operand's flag and extra_info
    assert len(both) == len(sintel) + len(kitti) and both.flow_list[len(sintel):] == kitti.flow_list
    three = 3 * kitti
    assert three.image_list == kitti.image_list * 3 and three.extra_info == kitti.extra_info
    gen = kitti()
    items = [next(gen) for _ in range(len(kitti) + 2)]                         # a training dataset wraps around
    np.testing.assert_array_equal(items[len(kitti)][0], items[0][0])
    assert sum(1 for _ in ds['kitti_test']()) == len(ds['kitti_test'])        # a test dataset ends
    np.random.seed(7)
    perm = np.random.permutation(len(kitti))
    shuffled = 1 * kitti
    np.random.seed(7)
    shuffled.shuffle()
    assert shuffled.flow_list == [kitti.flow_list[i] for i in perm]


@pytest.mark.parametrize('little', [True, False])
@pytest.mark.parametrize('color', [True, False])
def test_read_pfm(tmp_path, little, color):
    rng = np.random.default_rng(int(little) * 2 + int(color))
    data = rng.normal(0, 10, (3, 5, 3) if color else (3, 5)).astype(np.float32)
    path = str(tmp_path / 'x.pfm')
    write_pfm(path, data, little)
    got = frame_utils.read_pfm(path)
    np.testing.assert_array_equal(got, data)
    gen = frame_utils.read_gen(path)
    assert gen.dtype == np.float32
    np.testing.assert_array_equal(gen, data[..., :2] if color else data)
    bad = str(tmp_path / 'bad.pfm')
    open(bad, 'wb').write(b'P6\n5 3\n-1.0\n')
    with pytest.raises(ValueError, match='not a PFM'):
        frame_utils.read_pfm(bad)


def test_read_gen_dispatch(tmp_path):
    arr = np.arange(6, dtype=np.float64).reshape(2, 3)
    np.save(str(tmp_path / 'a.npy'), arr)
    os.rename(str(tmp_path / 'a.npy'), str(tmp_path / 'a.bin'))
    np.testing.assert_array_equal(frame_utils.read_gen(str(tmp_path / 'a.bin')), arr)
    flow = np.ones((2, 3, 2), np.float32)
    frame_utils.write_flow(str(tmp_path / 'f.flo'), flow)
    np.testing.assert_array_equal(frame_utils.read_gen(str(tmp_path / 'f.flo')), flow)
    assert frame_utils.read_gen(str(tmp_path / 'x.txt')) == []


def test_inflate_png16_checks_on_the_host(tmp_path):
    path = str(tmp_path / 'f.png')
    frame_utils.write_flow_kitti(path, np.zeros((3, 4, 2), np.float32))
    rows, h, w = frame_utils.inflate_png16(path)
    assert (h, w) == (3, 4) and len(rows) == 3 * (1 + 24)
    raw = open(path, 'rb').read()
    cut = str(tmp_path / 'cut.png')
    open(cut, 'wb').write(raw[:len(raw) - 20])
    with pytest.raises(ValueError, match='cut.png'):
        frame_utils.inflate_png16(cut)
    frame_utils.write_png(str(tmp_path / 'rgb8.png'), np.zeros((2, 2, 3), np.uint8))
    with pytest.raises(ValueError, match='rgb8.png.*16-bit'):
        frame_utils.inflate_png16(str(tmp_path / 'rgb8.png'))
    # an unknown filter byte, with a valid zlib stream around it
    import zlib
    body = bytearray(zlib.decompress(_idat(raw)))
    body[1 + 24] = 7
    bad = str(tmp_path / 'filter.png')
    open(bad, 'wb').write(_png16(bytes(body), 4, 3))
    with pytest.raises(ValueError, match='filter.png.*filter type 7 in row 1'):
        frame_utils.inflate_png16(bad)


def _idat(raw):
    return b''.join(body for kind, body in frame_utils._png_chunks(raw) if kind == b'IDAT')


def _png16(rows, w, h):
    import zlib

    def chunk(kind, body):
        return struct.pack('>I', len(body)) + kind + body + struct.pack('>I', zlib.crc32(kind + body) & 0xffffffff)
    return (b'\x89PNG\r\n\x1a\n' + chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, 16, 2, 0, 0, 0)) +
            chunk(b'IDAT', zlib.compress(rows)) + chunk(b'IEND', b''))


def test_metric_aggregations_match_numpy():
    from tf_raft_b200.evaluation import aggregate
    rng = np.random.default_rng(5)
    n = rng.integers(0, 50, 9)
    n[4] = 0
    c = np.stack([n] + [rng.integers(0, n + 1) for _ in range(4)], axis=1).astype(np.int64)
    s = rng.random(9) * n * 3
    sizes = [3, 2, 4]
    pix = aggregate(c, s, sizes, 'pixel')
    assert pix['epe'] == s.sum() / n.sum() and pix['u3'] == c[:, 2].sum() / n.sum()
    assert pix['fl_all'] == 100 * (c[:, 4].sum() / n.sum()) and pix['pixels'] == n.sum()
    img = aggregate(c[n > 0], s[n > 0], [int((n > 0).sum())], 'image')
    assert img['epe'] == np.mean(s[n > 0] / n[n > 0]) and img['u1'] == c[n > 0, 1].sum() / n.sum()
    assert np.isnan(aggregate(c, s, sizes, 'image')['epe'])                    # an empty image: NaN, as its mean
    ker = aggregate(c, s, sizes, 'keras')
    bounds = np.cumsum([0] + sizes)
    want = np.mean([s[a:b].sum() / n[a:b].sum() for a, b in zip(bounds[:-1], bounds[1:])])
    assert ker['epe'] == want
    want = np.mean([100 * (c[a:b, 4].sum() / n[a:b].sum()) for a, b in zip(bounds[:-1], bounds[1:])])
    assert ker['fl_all'] == want
    assert np.isnan(aggregate(np.zeros((1, 5), np.int64), np.zeros(1), [1], 'pixel')['epe'])
    with pytest.raises(ValueError, match='protocol'):
        aggregate(c, s, sizes, 'median')
