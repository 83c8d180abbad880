"""RAFT's evaluation padding on the host: InputPadder's offsets against RAFT's formula, `placement`, argument errors,
the scene split of the sequence loader, KITTI clamping, and raft_b200_pad_batch's host-side checks.  No GPU needed."""
import ctypes
import os

import numpy as np
import pytest
import torch

from tf_raft_b200.preprocess import InputPadder, _offsets, input_padding, placement

SIZES = [(436, 1024), (375, 1242), (370, 1224), (376, 1241), (1080, 2560)]      # Sintel, KITTI, HD1K


def _raft(h, w, mode):
    """RAFT core/utils/utils.py InputPadder.__init__, as stated: [left, right, top, bottom]."""
    pad_ht = (((h // 8) + 1) * 8 - h) % 8
    pad_wd = (((w // 8) + 1) * 8 - w) % 8
    if mode == 'sintel':
        return [pad_wd // 2, pad_wd - pad_wd // 2, pad_ht // 2, pad_ht - pad_ht // 2]
    return [pad_wd // 2, pad_wd - pad_wd // 2, 0, pad_ht]


@pytest.mark.parametrize('mode', ['sintel', 'kitti'])
def test_offsets_match_raft(mode):
    for h, w in [(h, w) for h in range(1, 65) for w in range(1, 65)] + SIZES:
        top, bottom, left, right = input_padding(h, w, mode)
        assert [left, right, top, bottom] == _raft(h, w, mode), (h, w)
        p = InputPadder((2, h, w, 3), mode)
        H, W = p.padded_size
        assert H % 8 == 0 and W % 8 == 0 and H - h < 8 and W - w < 8
        assert (H, W) == (-(-h // 8) * 8, -(-w // 8) * 8)          # what pad_to_multiple / target_size=None pick
        if h % 8 == 0 and w % 8 == 0:
            assert (top, bottom, left, right) == (0, 0, 0, 0)
        # the loader's placement of the frame in that padded size is the padder's
        assert placement(h, w, H, W, mode) == (top, left)
    assert InputPadder((1, 436, 1024, 3)).padded_size == (440, 1024)
    assert InputPadder((1, 375, 1242, 3), 'kitti').padded_size == (376, 1248)


def test_placement_crops_as_tf_and_pads_kitti_at_the_bottom():
    for size in range(1, 40):
        for target in range(1, 40):
            crop, pad = _offsets(size, target)
            for mode in ('sintel', 'kitti'):
                top, left = placement(size, size, target, target, mode)
                assert left == (-crop if crop else pad)
                assert top == (-crop if crop else (0 if mode == 'kitti' else pad))


def test_unpad_inverts_the_padding():
    """The host restatement of the kernel (np.pad 'edge' at the padder's offsets), then `unpad`, gives x back."""
    rng = np.random.default_rng(0)
    for mode in ('sintel', 'kitti'):
        for h, w in [(1, 1), (5, 7), (61, 84), (64, 96)]:
            x = rng.integers(0, 256, (2, h, w, 3)).astype(np.uint8)
            p = InputPadder(x.shape, mode)
            top, bottom, left, right = input_padding(h, w, mode)
            padded = torch.from_numpy(np.pad(x, ((0, 0), (top, bottom), (left, right), (0, 0)), mode='edge'))
            assert tuple(padded.shape[1:3]) == p.padded_size
            assert torch.equal(p.unpad(padded), torch.from_numpy(x))


def test_argument_errors():
    with pytest.raises(ValueError, match='pad mode'):
        InputPadder((1, 8, 8, 3), mode='chairs')
    with pytest.raises(ValueError, match='pad mode'):
        input_padding(8, 8, 'middlebury')
    with pytest.raises(ValueError):
        InputPadder((8, 8))
    p = InputPadder((1, 6, 6, 3))
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        p.pad(torch.zeros(1, 6, 6, 3, dtype=torch.uint8))
    from tf_raft_b200.datasets.dataset import FlowDataset, _check_padding
    with pytest.raises(ValueError, match='cannot crop'):
        FlowDataset._padded((60, 90), (56, 100), 'replicate')
    assert FlowDataset._padded((60, 90), (64, 96), 'replicate') == (64, 96)
    assert FlowDataset._padded((60, 90), (56, 100), 'zero') == (56, 100)
    with pytest.raises(ValueError, match='padding'):
        _check_padding('reflect', 'sintel')
    with pytest.raises(ValueError, match='pad_mode'):
        _check_padding('replicate', 'chairs')
    ds = FlowDataset()
    with pytest.raises(ValueError, match='padding'):
        next(ds.batches(1, padding='edge'))
    with pytest.raises(ValueError, match='pad_mode'):
        next(ds.sequences(pad_mode='bottom'))


def _touch(path):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    open(path, 'wb').close()


def test_scenes_need_chained_items(tmp_path):
    from tf_raft_b200 import datasets as D
    root = str(tmp_path / 'sintel')
    for scene, n in (('alley_1', 4), ('cave_4', 2), ('market_2', 3)):
        for i in range(n):
            _touch(os.path.join(root, 'test', 'clean', scene, 'frame_%04d.png' % (i + 1)))
    ds = D.MpiSintel(split='test', root=root)
    runs = ds.scenes()
    assert sorted(n for _, n in runs) == [1, 2, 3] and sum(n for _, n in runs) == len(ds)
    for i0, n in runs:
        assert len({ds.extra_info[k][0] for k in range(i0, i0 + n)}) == 1
        assert [ds.extra_info[k][1] for k in range(i0, i0 + n)] == list(range(n))
    shuffled = D.MpiSintel(split='test', root=root)          # what shuffle() does to a training split
    shuffled.image_list = shuffled.image_list[::-1]
    with pytest.raises(ValueError, match='do not chain'):
        shuffled.scenes()
    split = D.MpiSintel(split='test', root=root)
    i0, _ = next(r for r in runs if r[1] == 3)               # one item of that scene moved to the end
    split.image_list = split.image_list[:i0 + 1] + split.image_list[i0 + 2:] + [split.image_list[i0 + 1]]
    split.extra_info = split.extra_info[:i0 + 1] + split.extra_info[i0 + 2:] + [split.extra_info[i0 + 1]]
    with pytest.raises(ValueError, match='not one run|do not chain'):
        split.scenes()
    with pytest.raises(ValueError, match='extra_info'):
        (2 * ds).scenes()
    kroot = str(tmp_path / 'kitti')
    for i in range(3):
        for t in (10, 11):
            _touch(os.path.join(kroot, 'testing', 'image_2', '%06d_%d.png' % (i, t)))
    with pytest.raises(ValueError, match='extra_info'):
        D.KITTI(split='testing', root=kroot).scenes()
    chairs = D.FlowDataset()
    chairs.image_list = [['a.ppm', 'b.ppm'], ['c.ppm', 'd.ppm']]
    with pytest.raises(ValueError, match='extra_info'):
        chairs.scenes()
    broken = D.FlowDataset()
    broken.image_list = [['f1', 'f2'], ['f3', 'f4']]
    broken.extra_info = [('s', 0), ('s', 1)]
    with pytest.raises(ValueError, match='do not chain'):
        broken.scenes()


def test_kitti_flow_is_clamped_to_what_the_png_holds(tmp_path):
    from tf_raft_b200.datasets import frame_utils
    from tf_raft_b200.submission import KITTI_FLOW_MAX, KITTI_FLOW_MIN, kitti_flow_for_png
    flow = torch.tensor([[[-1e4, 1e4], [-512.0, 511.984375], [600.0, float('nan')],
                          [float('-inf'), float('inf')], [1.25, -3.5]]], dtype=torch.float32)
    got = kitti_flow_for_png(flow).numpy()
    want = np.array([[[-512, 511.984375], [-512, 511.984375], [511.984375, 0], [-512, 511.984375], [1.25, -3.5]]],
                    np.float32)
    assert np.array_equal(got, want)
    assert float(64.0 * np.float32(KITTI_FLOW_MIN) + 2 ** 15) == 0 and float(64.0 * np.float32(KITTI_FLOW_MAX) + 2 ** 15) == 65535
    path = str(tmp_path / 'f.png')
    frame_utils.write_flow_kitti(path, got)
    back, valid = frame_utils.read_flow_kitti(path)
    assert np.array_equal(back, want) and np.all(valid == 1)


@pytest.fixture(scope='module')
def L():
    from tf_raft_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_pad_batch_host_side_errors(L):
    """raft_b200_pad_batch checks every plane on the host and launches nothing on a bad one (no device needed: the
    pointers below are never dereferenced)."""
    from tf_raft_b200.preprocess import _PadPlane

    def plane(**kw):
        p = _PadPlane(src=0x1000, dst=0x2000, h=4, w=5, c=3, H=8, W=8, top=2, left=1, dtype=0, mode=1)
        for k, v in kw.items():
            setattr(p, k, v)
        return p

    def call(*planes, n=None, dev=0x3000):
        arr = (_PadPlane * len(planes))(*planes)
        return L.raft_b200_pad_batch(arr, ctypes.c_void_p(dev), len(planes) if n is None else n, None)

    assert call(plane(), dev=None) == -1                    # no device array
    assert L.raft_b200_pad_batch(None, ctypes.c_void_p(0x3000), 1, None) == -1
    assert call(plane(), n=0) == -2
    assert call(plane(src=None)) == -1
    assert call(plane(dst=None)) == -1
    assert call(plane(dtype=2)) == -1                       # unknown dtype
    assert call(plane(mode=5)) == -1                        # unknown mode
    assert call(plane(dtype=1, src=0x1002)) == -1           # float32 plane not 4-byte aligned
    assert call(plane(dtype=1, dst=0x2001)) == -1
    assert call(plane(h=0)) == -2
    assert call(plane(W=0)) == -2
    assert call(plane(c=0)) == -2
    assert call(plane(H=1 << 16, W=1 << 15)) == -2          # H * W * c beyond 2^31 - 1
    assert call(plane(), plane(h=-1)) == -2                 # any plane of the batch
    big = (_PadPlane * 1)(plane())
    assert L.raft_b200_pad_batch(big, ctypes.c_void_p(0x3000), 65536, None) == -2
