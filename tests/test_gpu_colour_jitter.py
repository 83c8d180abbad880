"""GPU: colour='torchvision' (raft_b200_colour_jitter, csrc/colour.cuh) byte for byte.  Each op against the NumPy
restatement of Pillow (oracle/pil_colour_np.py) over all 2^24 colours; contrast's degenerate images; both augmentors end
to end against the original RAFT's augmentors on the real torchvision, PIL and cv2 (oracle/raft_augment.py) at Chairs,
Sintel, KITTI and HD1K sizes, stacked and asymmetric, in every op order; mixed-size batches, FlowDataset.batches and
repeat runs; RAFT's --add_noise; and scripts/train.py with both new options.
"""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import pil_colour_np as P

pytestmark = pytest.mark.gpu
R = pytest.importorskip('oracle.raft_augment', reason='the RAFT oracle needs torchvision, Pillow and OpenCV')

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
# (kind, source size, RAFT's augmentor arguments at that dataset's stage, core/datasets.py fetch_dataloader)
SIZES = {
    'chairs': ('dense', (384, 512), dict(crop_size=(368, 496), min_scale=-0.1, max_scale=1.0, do_flip=True)),
    'sintel': ('dense', (436, 1024), dict(crop_size=(368, 768), min_scale=-0.2, max_scale=0.6, do_flip=True)),
    'kitti': ('sparse', (375, 1242), dict(crop_size=(288, 960), min_scale=-0.2, max_scale=0.4, do_flip=False)),
    'hd1k': ('sparse', (1080, 2560), dict(crop_size=(368, 768), min_scale=-0.5, max_scale=0.2, do_flip=True)),
}


@pytest.fixture(scope='module')
def D():
    from tf_raft_b200 import _lib, build
    import tf_raft_b200.datasets as datasets
    build.build()
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    return datasets


def _cls(D, kind):
    return D.FlowAugmentor if kind == 'dense' else D.SparseFlowAugmentor


def _sample(rng, h, w, sparse=False):
    img1 = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    img2 = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    img1[: h // 4] = img1[: h // 4, :1]                              # greys and smooth rows
    img2[h // 2: h // 2 + h // 8] = img2[h // 2: h // 2 + h // 8, :1]
    flow = (rng.standard_normal((h, w, 2)) * 20).astype(np.float32)
    if not sparse:
        return img1, img2, flow
    return img1, img2, flow, (rng.uniform(size=(h, w)) < 0.3).astype(np.float32)


def _cuda(sample):
    return tuple(torch.from_numpy(a).cuda() for a in sample)


def _jitter_only(D, img1, img2, jitter):
    """The augmentor with nothing but the jitter: full-size crop, no eraser, no resize or flip."""
    h, w = img1.shape[:2]
    p = D.AugmentParams((None, None), (None, None), [], 1.0, 1.0, False, False, False, 0, 0, (h, w), jitter)
    out = D.FlowAugmentor((h, w)).batch([_cuda((img1, img2, np.zeros((h, w, 2), np.float32)))], [p])
    return out[0][0].cpu().numpy(), out[1][0].cpu().numpy()


def _want_jitter(img1, img2, jitter):
    if len(jitter) == 1:
        (order, b, c, s, h), = jitter
        return tuple(np.split(P.jitter(np.concatenate([img1, img2]), order, (b, c, s), h), 2))
    return tuple(P.jitter(x, j[0], j[1:4], j[4]) for x, j in zip((img1, img2), jitter))


def _assert_same(got, want, what):
    for k, (g, w) in enumerate(zip(got, want)):
        if not np.array_equal(g, w):
            bad = np.argwhere(g != w)
            raise AssertionError(f'{what}: output {k}: {len(bad)} bytes differ, first at {bad[0].tolist()}: '
                                 f'{g[tuple(bad[0])]} vs {w[tuple(bad[0])]}')


# ------------------------------------------------------------------------------------------------ each op
def _all_colours():
    c = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)


OP_CASES = [
    ('brightness', (0, 1, 2, 3), (0.6, None, None, None)), ('brightness', (0, 1, 2, 3), (1.4, None, None, None)),
    ('brightness', (0, 1, 2, 3), (1.0 + 2.0 ** -23, None, None, None)),
    ('contrast', (1, 0, 2, 3), (None, 0.6, None, None)), ('contrast', (1, 0, 2, 3), (None, 1.3999999761581, None, None)),
    ('saturation', (2, 1, 0, 3), (None, None, 0.6137, None)), ('saturation', (2, 1, 0, 3), (None, None, 1.4, None)),
    ('hue', (3, 1, 2, 0), (None, None, None, 0.159)), ('hue', (3, 1, 2, 0), (None, None, None, -0.159)),
    ('hue', (3, 1, 2, 0), (None, None, None, 0.003)), ('hue', (3, 1, 2, 0), (None, None, None, 0.0)),
]


@pytest.mark.parametrize('name,order,factors', OP_CASES, ids=[f'{c[0]}-{i}' for i, c in enumerate(OP_CASES)])
def test_each_op_every_colour(D, name, order, factors):
    """One op over all 2^24 colours (one 4096 x 4096 image) as img1, and over the same colours reversed as img2 with
    its own set; contrast also with both images as one stacked set, whose grey is their common mean."""
    img1 = _all_colours()
    img2 = np.ascontiguousarray(img1[::-1, ::-1])
    draws = (order, *[None if f is None else float(np.float32(f)) for f in factors])
    second = ((2, 3, 0, 1),) + tuple(None if f is None else float(np.float32(f * 0.9)) for f in draws[1:])
    for jitter in ((draws, second), (draws,)) if name == 'contrast' else ((draws, second),):
        _assert_same(_jitter_only(D, img1, img2, jitter), _want_jitter(img1, img2, jitter), f'{name} {jitter}')


def test_degenerate_images(D):
    """Constant, black and white images, where contrast's grey is the image itself, in all four ops' orders."""
    rng = np.random.default_rng(3)
    for v1, v2 in ((0, 0), (255, 255), (0, 255), (128, 128), (37, 200)):
        img1, img2 = np.full((64, 80, 3), v1, np.uint8), np.full((64, 80, 3), v2, np.uint8)
        img1[0, 0] = (v1, 255 - v1, v1)                          # one coloured pixel so that hue has work
        for order in ((0, 1, 2, 3), (1, 3, 2, 0), (3, 2, 1, 0)):
            b, c, s = (float(np.float32(x)) for x in rng.uniform(0.6, 1.4, 3))
            h = float(np.float32(rng.uniform(-0.16, 0.16)))
            for jitter in (((order, b, c, s, h),), ((order, b, c, s, h), (order[::-1], c, b, s, -h))):
                _assert_same(_jitter_only(D, img1, img2, jitter), _want_jitter(img1, img2, jitter),
                             f'{v1}/{v2} {jitter}')


# ------------------------------------------------------------------------------------------------ end to end
def _oracle(kind, aug_args, sample):
    cls = R.FlowAugmentor if kind == 'dense' else R.SparseFlowAugmentor
    return cls(**aug_args)(*[a.copy() for a in sample])


def _compare(kind, got, want, what):
    """GPU (img1, img2, flow, valid) against RAFT's output: images bytes, flow float32 bits, valid -- dense: |flow| <
    1000 on RAFT's float64 flow (the project's dense valid), sparse: RAFT's valid."""
    flow = want[2].astype(np.float32)
    valid = ((np.abs(want[2][..., 0]) < 1000) & (np.abs(want[2][..., 1]) < 1000)) if kind == 'dense' else want[3]
    _assert_same(got[:2], want[:2], what)
    assert np.array_equal(got[2].view(np.uint32), flow.view(np.uint32)), f'{what}: flow'
    assert np.array_equal(got[3], valid.astype(np.float32)), f'{what}: valid'


def _run(D, kind, aug_args, samples, seeds):
    """Draw each sample's parameters under its (np, torch) seeds, augment them as one GPU batch, and compare each with
    RAFT's augmentor run under the same seeds; returns the parameters."""
    aug = _cls(D, kind)(colour='torchvision', **aug_args)
    params = []
    for s, (ns, ts) in zip(samples, seeds):
        np.random.seed(ns)
        torch.manual_seed(ts)
        params.append(aug.sample_params(*s[0].shape[:2]))
    got = [t.cpu().numpy() for t in aug.batch([_cuda(s) for s in samples], params)]
    for i, (s, (ns, ts)) in enumerate(zip(samples, seeds)):
        np.random.seed(ns)
        torch.manual_seed(ts)
        want = _oracle(kind, aug_args, s)
        _compare(kind, [g[i] for g in got], want, f'{kind} sample {i} seeds {(ns, ts)} params {params[i]}')
    return params


def _np_seeds(n, asym=None):
    out, seed = [], 0
    while len(out) < n:
        np.random.seed(seed)
        if asym is None or (np.random.rand() < 0.2) == asym:
            out.append(seed)
        seed += 1
    return out


@pytest.mark.parametrize('name', sorted(SIZES))
def test_seeded_against_raft(D, name):
    kind, (h, w), aug_args = SIZES[name]
    rng = np.random.default_rng(7)
    seeds = list(zip(_np_seeds(2, False) + (_np_seeds(2, True) if kind == 'dense' else _np_seeds(1)), range(10, 20)))
    samples = [_sample(rng, h, w, kind == 'sparse') for _ in seeds]
    params = _run(D, kind, aug_args, samples, seeds)
    assert {len(p.jitter) for p in params} == ({1, 2} if kind == 'dense' else {1})
    print(name, [(p.jitter, p.spatial, len(p.rects)) for p in params])


def _torch_seed_for(order):
    for seed in range(100000):
        torch.manual_seed(seed)
        if tuple(int(i) for i in torch.randperm(4)) == order:
            return seed
    raise AssertionError(order)


@pytest.mark.parametrize('name', ['chairs', 'kitti'])
def test_every_op_order_against_raft(D, name):
    """All 24 orders in one batch, each drawn by RAFT's own stream (a torch seed whose randperm gives it); dense
    samples alternate stacked and asymmetric gates."""
    kind, (h, w), aug_args = SIZES[name]
    rng = np.random.default_rng(8)
    orders = list(itertools.permutations(range(4)))
    stacked, asym = _np_seeds(24, False), _np_seeds(12, True)
    np_seeds = [asym[i // 2] if kind == 'dense' and i % 2 else stacked[i] for i in range(24)]
    seeds = list(zip(np_seeds, [_torch_seed_for(o) for o in orders]))
    samples = [_sample(rng, h, w, kind == 'sparse') for _ in orders]
    params = _run(D, kind, aug_args, samples, seeds)
    assert sorted(p.jitter[0][0] for p in params) == orders


def test_narrow_images(D):
    """Below ~24 output columns the kernels' resize differs from cv2's scalar row tail (oracle/augment_np.py), with
    either colour step: there the GPU equals RAFT's jitter followed by the project's resize restatement."""
    from oracle import augment_np as A
    rng = np.random.default_rng(9)
    img1, img2, flow = _sample(rng, 40, 20)
    torch.manual_seed(4)
    jitter = (D.augmentor.jitter_params(0.4, 0.4, 0.4, 0.5 / 3.14),)
    j1, j2 = _raft_jitter(img1, img2, jitter)
    _assert_same(_jitter_only(D, img1, img2, jitter), (j1, j2), 'narrow jitter')
    p = D.AugmentParams((None, None), (None, None), [], 0.9, 1.1, True, True, False, 1, 2, (30, 12), jitter)
    got = [t[0].cpu().numpy() for t in D.FlowAugmentor((30, 12)).batch([_cuda((img1, img2, flow))], [p])]
    want = A.augment_dense(j1, j2, flow, p)
    _assert_same(got[:2], want[:2], 'narrow images')
    assert np.array_equal(got[2].view(np.uint32), want[2].view(np.uint32))


def _raft_jitter(img1, img2, jitter):
    aug = R.FlowAugmentor((8, 8))
    aug.photo_aug = R.ReplayJitter(jitter)
    if len(jitter) == 2:
        return R._jitter(aug.photo_aug, img1), R._jitter(aug.photo_aug, img2)
    return tuple(np.split(R._jitter(aug.photo_aug, np.concatenate([img1, img2])), 2))


# ------------------------------------------------------------------------------------------------ batching
def test_mixed_batch_equals_one_by_one_and_repeats(D):
    rng = np.random.default_rng(10)
    aug = D.FlowAugmentor((368, 496), colour='torchvision')
    shapes = [(384, 512), (436, 1024), (401, 611), (384, 512), (436, 1024)]
    samples = [_sample(rng, *s) for s in shapes]
    np.random.seed(31)
    torch.manual_seed(32)
    params = [aug.sample_params(*s) for s in shapes]
    got = [t.cpu() for t in aug.batch([_cuda(s) for s in samples], params)]
    again = [t.cpu() for t in aug.batch([_cuda(s) for s in samples], params)]
    assert all(torch.equal(a, b) for a, b in zip(got, again))
    for i, (s, p) in enumerate(zip(samples, params)):
        one = aug(*_cuda(s), params=p)
        for k in range(3):
            assert torch.equal(one[k].cpu(), got[k][i]), (i, k)


def test_flow_dataset_batches_equal_items(D, tmp_path):
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import test_gpu_fit as gf
    data, split = gf._write_chairs(str(tmp_path))
    args = dict(gf.AUG, colour='torchvision')

    def dataset():
        np.random.seed(5)
        torch.manual_seed(6)
        return D.FlyingChairs(args, split='training', split_txt=split, root=data)

    ds = dataset()
    batched = [[t.cpu() for t in b] for b in ds.batches(2, workers=2)]
    ds = dataset()
    items = [[t.cpu() for t in ds[i]] for i in range(len(ds))]
    assert ds.augmentor.colour == 'torchvision'
    flat = [[b[k][j] for k in range(4)] for b in batched for j in range(b[0].shape[0])]
    assert len(flat) == len(items)
    for i, (a, b) in enumerate(zip(flat, items)):
        assert all(torch.equal(x, y) for x, y in zip(a, b)), i


# ------------------------------------------------------------------------------------------------ add_noise
def test_add_noise_is_rafts(D):
    rng = np.random.default_rng(11)
    im1 = torch.from_numpy(rng.integers(0, 256, (2, 96, 128, 3), dtype=np.uint8)).cuda()
    im2 = torch.from_numpy(rng.integers(0, 256, (2, 96, 128, 3), dtype=np.uint8)).cuda()
    for seed in (0, 3):
        np.random.seed(seed)
        torch.manual_seed(seed + 100)
        got = D.add_noise(im1, im2)
        np.random.seed(seed)
        torch.manual_seed(seed + 100)
        image1, image2 = (x.permute(0, 3, 1, 2).float() for x in (im1, im2))        # RAFT's NCHW float batch
        stdv = np.random.uniform(0.0, 5.0)
        image1 = (image1 + stdv * torch.randn(*image1.shape).cuda()).clamp(0.0, 255.0)
        image2 = (image2 + stdv * torch.randn(*image2.shape).cuda()).clamp(0.0, 255.0)
        for g, w in zip(got, (image1, image2)):
            assert g.dtype == torch.float32 and g.is_contiguous()
            assert torch.equal(g, w.permute(0, 2, 3, 1)), seed
        assert not torch.equal(got[0], im1.float())


# ------------------------------------------------------------------------------------------------ the script
def test_train_script_with_torchvision_colour_and_noise(D, tmp_path):
    yaml = pytest.importorskip('yaml', reason='scripts/train.py reads YAML configs and needs PyYAML')
    from oracle import raft_pytorch as rp
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import test_gpu_fit as gf
    data, split = gf._write_chairs(str(tmp_path / 'chairs'))
    src = tmp_path / 'raft-synthetic.pth'
    torch.save(rp.synthetic_checkpoint(seed=11), src)
    config = {'data': {'root': data, 'split_txt': split}, 'augment': gf.AUG,
              'model': {'iters': 2, 'iters_pred': 2, 'resume': 0},
              'train': {'epochs': 1, 'batch_size': gf.BATCH, 'learning_rate': 1e-4, 'weight_decay': 1e-5,
                        'clip_norm': 1.0},
              'visualize': {'num_visualize': 1, 'choose_random': False}, 'logdir': str(tmp_path / 'logs')}
    cfg = str(tmp_path / 'run.yml')
    with open(cfg, 'w') as f:
        yaml.dump(config, f)
    proc = subprocess.run([sys.executable, os.path.join(ROOT, 'scripts', 'train.py'), 'chairs', cfg, '--workers', '2',
                           '--pytorch-checkpoint', str(src), '--colour-jitter', 'torchvision', '--add-noise',
                           '--seed', '1'], capture_output=True, text=True, timeout=1200)
    assert proc.returncode == 0, proc.stdout[-3000:] + proc.stderr[-3000:]
    assert 'wrote' in proc.stdout and os.path.exists(proc.stdout.split('wrote ')[-1].split()[0])
