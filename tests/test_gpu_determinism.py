"""Reproducible training on one GPU.

The lookup backward and SmallRAFT's upsampling backward add their terms in a fixed order, stated in
tf_raft_b200/csrc/train.cuh, kernels.cuh and include/raft_b200.h.  The first two tests hold each kernel to the NumPy
float32 emulation of that order (oracle/determinism_np.py) bit for bit; that is the proof.  The rest are consequences:
the same train_step from the same state gives the same bits, training runs under torch.use_deterministic_algorithms,
and fit, a save/load resume and scripts/train.py --seed reproduce their results exactly."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cases
from oracle import determinism_np as dn, weights
from test_determinism_ref import KINDS, LOOKUP_CONFIGS, lookup_pyramid

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def assert_bits(got, want, what):
    """NaN at the same places, every other element the same bits."""
    got = np.ascontiguousarray(got, dtype=np.float32)
    want = np.ascontiguousarray(want, dtype=np.float32)
    assert got.shape == want.shape, what
    nan_g, nan_w = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan_g, nan_w), f'{what}: NaN at {int((nan_g != nan_w).sum())} other places'
    diff = got.view(np.int32)[~nan_g] != want.view(np.int32)[~nan_w]
    assert not diff.any(), f'{what}: {int(diff.sum())} of {diff.size} differ, max-abs ' \
                           f'{float(np.abs(got[~nan_g] - want[~nan_w]).max()):.3e}'


def gpu_lookup_backward(pyr, coords, g, radius, gc_in, gp_in):
    """raft_b200_corr_lookup_backward accumulating into copies of gc_in / gp_in."""
    from tf_raft_b200 import _lib
    nq = coords.reshape(-1, 2).shape[0]
    b, h, w = coords.shape[:3]
    P = [dev(p) for p in pyr]
    c, go = dev(coords), dev(g)                  # held until the call has run: a freed buffer could be handed out again
    gc = dev(gc_in)
    gp = [dev(x) for x in gp_in]
    _lib.call('corr_lookup_backward', gc.device, _lib.ptr_array(P), _lib.ptr(c), _lib.ptr(go), b, h, w,
              len(P), radius, _lib.ptr(gc), _lib.ptr_array(gp))
    torch.cuda.synchronize()
    return gc.cpu().numpy().reshape(nq, 2), [x.cpu().numpy().reshape(nq, *p.shape[1:3]) for x, p in zip(gp, pyr)]


def check_lookup(pyr, coords, g, radius, seed, what):
    nq = coords.reshape(-1, 2).shape[0]
    rng = np.random.default_rng(seed)
    gc_in = rng.standard_normal((nq, 2)).astype(np.float32)
    gp_in = [rng.standard_normal(p.shape[:3]).astype(np.float32) for p in pyr]
    got_c, got_p = gpu_lookup_backward(pyr, coords, g, radius, gc_in, gp_in)
    want_c, want_p = dn.lookup_backward(pyr, coords, g, radius, gc_in, gp_in)
    assert_bits(got_c, want_c, f'{what}: grad_coords')
    for l, (a, e) in enumerate(zip(got_p, want_p)):
        assert_bits(a, e, f'{what}: grad_pyr[{l}]')


# --------------------------------------------------------------------------------------------- 1. lookup backward
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('radius,levels', LOOKUP_CONFIGS)
def test_lookup_backward_equals_the_emulation(radius, levels, kind):
    """Every grid of cases.LOOKUP_GRIDS, with non-zero accumulators on entry, bit for bit."""
    for b, h, w in cases.LOOKUP_GRIDS[levels]:
        pyr = lookup_pyramid(b, h, w, levels)
        coords = cases.lookup_coords(b, h, w, kind)
        g = np.random.default_rng(5).standard_normal((b, h, w, levels * (2 * radius + 1) ** 2)).astype(np.float32)
        g[..., ::13] = 0                                           # skipped taps
        check_lookup(pyr, coords, g, radius, 11 + h, f'r={radius} levels={levels} {b}x{h}x{w} {kind}')


@pytest.mark.parametrize('radius,levels', [(4, 4), (3, 4), (5, 6)])
def test_lookup_backward_equals_the_emulation_with_non_finite_operands(radius, levels):
    """NaN and +-inf planted in grad_out, in the coordinates and in the pyramid: the same NaN cells and the same bits
    elsewhere."""
    b, h, w = cases.LOOKUP_GRIDS[levels][0]
    pyr = lookup_pyramid(b, h, w, levels)
    coords = cases.lookup_coords(b, h, w, 'jitter')
    ntap = (2 * radius + 1) ** 2
    g = np.random.default_rng(8).standard_normal((b, h, w, levels * ntap)).astype(np.float32)
    rng = np.random.default_rng(9)
    nq = b * h * w
    gf, cf = g.reshape(nq, -1), coords.reshape(nq, 2)
    for v in (np.nan, np.inf, -np.inf):
        gf[rng.integers(0, nq, 3), rng.integers(0, levels * ntap, 3)] = v
        cf[rng.integers(0, nq, 2), rng.integers(0, 2, 2)] = v
        for p in pyr:
            p.reshape(nq, -1)[rng.integers(0, nq, 4), rng.integers(0, p[0].size, 4)] = v
    check_lookup(pyr, coords, g, radius, 12, f'r={radius} levels={levels} non-finite')


def chairs_lookup_case(b=4, h=46, w=62, seed=0):
    """The Chairs training grid (368 x 496 images), a random 4-level pyramid and the coordinates of a smooth flow of a
    few pixels with sub-pixel detail, as in the middle of training."""
    rng = np.random.default_rng(seed)
    pyr = [rng.standard_normal((b * h * w, h >> l, w >> l, 1)).astype(np.float32) for l in range(4)]
    gy, gx = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing='ij')
    fx = 6 * np.sin(gy / 9 + 0.3) + 3 * np.cos(gx / 13) + rng.normal(0, 0.4, (b, h, w))
    fy = 4 * np.cos(gx / 11 - 0.2) - 2 * np.sin(gy / 7) + rng.normal(0, 0.4, (b, h, w))
    coords = np.stack([gx + fx, gy + fy], axis=-1).astype(np.float32)
    return pyr, coords


def test_lookup_backward_equals_the_emulation_at_the_chairs_training_shape():
    pyr, coords = chairs_lookup_case()
    g = (np.random.default_rng(1).standard_normal(coords.shape[:3] + (4 * 81,)) * 1e-3).astype(np.float32)
    check_lookup(pyr, coords, g, 4, 13, 'Chairs 4x46x62 r=4')


# --------------------------------------------------------------------------------------------- 2. upsampling backward
def gpu_upflow8_backward(g):
    from tf_raft_b200 import _lib
    b, H, W, _ = g.shape
    gd = dev(g)
    out = torch.full((b, H // 8, W // 8, 2), 7.0, device='cuda')
    _lib.call('upflow8_backward', gd.device, _lib.ptr(gd), b, H // 8, W // 8, _lib.ptr(out))
    return out.cpu().numpy()


@pytest.mark.parametrize('shape', [(4, 46, 62), (8, 46, 62), (2, 55, 61), (3, 9, 13), (1, 1, 6), (2, 4, 1), (1, 1, 1)],
                         ids=lambda s: 'x'.join(map(str, s)))
def test_upflow8_backward_equals_the_emulation(shape):
    """SmallRAFT's training shapes (batch 4, and 2B = 8 for the self-supervised step), odd sizes and h or w = 1."""
    b, h, w = shape
    g = np.random.default_rng(h + w).standard_normal((b, 8 * h, 8 * w, 2)).astype(np.float32)
    assert_bits(gpu_upflow8_backward(g), dn.upflow8_backward(g), f'upflow8 backward {shape}')


@pytest.mark.parametrize('shape', [(2, 5, 7), (1, 1, 6), (2, 4, 1)], ids=lambda s: 'x'.join(map(str, s)))
def test_upflow8_backward_nan_cells_match_torch(shape):
    b, h, w = shape
    H, W = 8 * h, 8 * w
    g = np.random.default_rng(4).standard_normal((b, H, W, 2)).astype(np.float32)
    for Y, X, v in ((0, 0, np.nan), (H - 1, W - 1, np.inf), (2, W - 3, np.nan), (H // 2, 1, -np.inf)):
        g[-1, Y, X, (Y + X) % 2] = v
    x = torch.zeros((b, 2, h, w), device='cuda', requires_grad=True)
    F.interpolate(x, scale_factor=8, mode='bilinear', align_corners=False).backward(dev(g).permute(0, 3, 1, 2))
    want = x.grad.permute(0, 2, 3, 1).cpu().numpy()
    got = gpu_upflow8_backward(g)
    assert np.isnan(want).any()
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert_bits(got, dn.upflow8_backward(g), f'upflow8 backward non-finite {shape}')


# --------------------------------------------------------------------------------------------- 3. the training step
def _model(variant, train_precision, unsup, seed=21):
    import tf_raft_b200 as T
    model = (T.RAFT if variant == 'raft' else T.SmallRAFT)(iters=2, iters_pred=2, precision='f16x2')
    model.load_params(weights.init_params(variant, seed, bias_scale=0.05, norm_jitter=0.1))
    kw = dict(loss=T.UnsupervisedLoss()) if unsup else {}
    model.compile(optimizer=T.AdamW(weight_decay=1e-4, learning_rate=T.CyclicalLearningRate(1e-4, 2e-4, 2)),
                  clip_norm=1.0, train_precision=train_precision, **kw)
    return model


def _batches(n, unsup):
    out = []
    for s in range(n):
        im1, im2 = (torch.from_numpy(a).cuda() for a in cases.images(2, 64, 96, 3 + s, 40 + s))
        rng = np.random.default_rng(s)
        flow = torch.from_numpy((rng.standard_normal((2, 64, 96, 2)) * 5).astype(np.float32)).cuda()
        valid = torch.from_numpy(rng.uniform(size=(2, 64, 96)) > 0.1).cuda()
        out.append((im1, im2) if unsup else (im1, im2, flow, valid))
    return out


def _state(model):
    t = model._trainer
    return dict(p=t.flat.p, g=t.flat.g, m=t.flat.m, v=t.flat.v, **t.moving)


@pytest.mark.parametrize('loss', ['sequence', 'unsupervised'])
@pytest.mark.parametrize('train_precision', ['fp32', 'f16x2'])
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_train_step_twice_gives_the_same_bits(variant, train_precision, loss):
    """Two models from the same seed, three train_steps each on the same batches: the losses, the flat parameters,
    gradients and Adam moments, and the moving statistics are identical."""
    unsup = loss == 'unsupervised'
    data = _batches(3, unsup)
    runs = []
    for _ in range(2):
        model = _model(variant, train_precision, unsup)
        losses = [float(model.train_step(d)['loss']) for d in data]
        runs.append((losses, {k: v.detach().cpu().clone() for k, v in _state(model).items()}))
        del model
    (la, sa), (lb, sb) = runs
    assert la == lb
    assert sorted(sa) == sorted(sb)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k


_DETERMINISTIC = r'''
import os, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], 'tests'))
import torch
torch.use_deterministic_algorithms(True)
import test_gpu_determinism as t
for unsup in (False, True):
    model = t._model(sys.argv[2], 'fp32', unsup)
    out = model.train_step(t._batches(1, unsup)[0])
    loss = float(out['loss'])
    assert loss == loss, 'NaN loss'
    assert all(bool(torch.isfinite(v).all()) for v in t._state(model).values()), 'non-finite state'
    print('OK', sys.argv[2], 'unsupervised' if unsup else 'sequence', loss)
'''


@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_train_step_runs_under_torch_deterministic_algorithms(variant):
    """One train_step per loss with torch.use_deterministic_algorithms(True), which raises for an op without a
    deterministic implementation and fills torch.empty with NaN (so a read of uninitialised memory shows)."""
    res = subprocess.run([sys.executable, '-c', _DETERMINISTIC, ROOT, variant], capture_output=True, text=True,
                         timeout=900, env={**os.environ, 'CUBLAS_WORKSPACE_CONFIG': ':4096:8',
                                           'PYTHONDONTWRITEBYTECODE': '1'})
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    assert res.stdout.count('OK ') == 2, res.stdout


# --------------------------------------------------------------------------------------------- 4. fit, resume, script
@pytest.fixture(scope='module')
def chairs(tmp_path_factory):
    import test_gpu_fit as gf
    return gf._write_chairs(str(tmp_path_factory.mktemp('chairs')))


def _trainer_state(model):
    t = model._trainer
    return dict(p=t.flat.p, m=t.flat.m, v=t.flat.v, **t.moving)


@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_fit_twice_and_a_resumed_fit_give_the_same_bits(chairs, tmp_path, variant):
    """fit with the same seeds twice: identical trainer state and byte-identical ModelCheckpoint files.  One epoch,
    save_weights, load_weights into a fresh model and a second epoch on the same batch stream: the uninterrupted
    run's state bit for bit."""
    import test_gpu_fit as gf
    from tf_raft_b200 import ModelCheckpoint
    states, files = [], []
    for run in range(2):
        model, _ = gf._model(variant)
        train, _ = gf._datasets(chairs, 5)
        ckpt = ModelCheckpoint(str(tmp_path / f'run{run}' / 'model-{epoch}'), save_weights_only=True)
        model.fit(train.batches(gf.BATCH, workers=2, repeat=True), epochs=gf.EPOCHS, steps_per_epoch=gf.STEPS,
                  callbacks=[ckpt], verbose=0)
        states.append({k: v.detach().cpu().clone() for k, v in _trainer_state(model).items()})
        files.append({os.path.relpath(p, tmp_path / f'run{run}'): open(p, 'rb').read()
                      for p in sorted(glob.glob(str(tmp_path / f'run{run}' / '*')))})
    for k in states[0]:
        assert torch.equal(states[0][k], states[1][k]), k
    assert len(files[0]) >= 2 * gf.EPOCHS and sorted(files[0]) == sorted(files[1])
    for name, data in files[0].items():
        assert data == files[1][name], name

    first, _ = gf._model(variant)
    train, _ = gf._datasets(chairs, 5)
    stream = train.batches(gf.BATCH, workers=2, repeat=True)
    first.fit(stream, epochs=1, steps_per_epoch=gf.STEPS, verbose=0)
    prefix = str(tmp_path / 'resume' / 'model')
    first.save_weights(prefix)
    second, _ = gf._model(variant, seed=99)
    second.load_weights(prefix)
    second.fit(stream, epochs=1, steps_per_epoch=gf.STEPS, verbose=0)
    assert second.optimizer.iterations == gf.EPOCHS * gf.STEPS
    resumed = _trainer_state(second)
    for k, v in states[0].items():
        assert torch.equal(resumed[k].cpu(), v), k


def test_train_script_with_a_seed_writes_the_same_checkpoint_twice(chairs, tmp_path):
    yaml = pytest.importorskip('yaml', reason='scripts/train.py reads YAML configs and needs PyYAML')
    import test_gpu_fit as gf
    data, split = chairs
    blobs = []
    for run in range(2):
        config = {'data': {'root': data, 'split_txt': split}, 'augment': gf.AUG,
                  'model': {'iters': 2, 'iters_pred': 2, 'resume': 0},
                  'train': {'epochs': 1, 'batch_size': gf.BATCH, 'learning_rate': 4e-4, 'weight_decay': 1e-4,
                            'clip_norm': 1},
                  'visualize': {'num_visualize': 1, 'choose_random': True}, 'logdir': str(tmp_path / f'logs{run}')}
        cfg = str(tmp_path / f'run{run}.yml')
        with open(cfg, 'w') as f:
            yaml.dump(config, f)
        proc = subprocess.run([sys.executable, os.path.join(ROOT, 'scripts', 'train.py'), 'chairs', cfg, '--seed', '3',
                               '--workers', '2'], capture_output=True, text=True, timeout=1200)
        assert proc.returncode == 0, proc.stdout[-3000:] + proc.stderr[-3000:]
        (logdir,) = glob.glob(os.path.join(config['logdir'], '*'))
        paths = sorted(glob.glob(os.path.join(logdir, 'checkpoints', 'model*')))
        assert paths
        blobs.append({os.path.basename(p): open(p, 'rb').read() for p in paths})
    assert sorted(blobs[0]) == sorted(blobs[1])
    for name, data in blobs[0].items():
        assert data == blobs[1][name], name
