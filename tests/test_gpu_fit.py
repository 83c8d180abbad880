"""`RAFT.fit`, `save_weights` / `load_weights`, `ModelCheckpoint` and `scripts/train.py` on the GPU, on a synthetic
FlyingChairs tree (96x128 .ppm pairs, .flo flows, a split file) with 64x96 crops.

The lookup backward scatters its gradient with fp32 atomicAdd (csrc/train.cuh), so two training runs on the same batches
are not bit-identical: a run through `fit` and the same steps by hand are compared within a tolerance, while what `fit`
feeds (batches, learning rates) and what a checkpoint holds are compared bit for bit."""
import glob
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import weights

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
H, W, CROP = 96, 128, (64, 96)                  # crops of 64 x 96: four pyramid levels down to 1 x 1
N_TRAIN, N_VAL, BATCH, STEPS, EPOCHS = 5, 2, 2, 3, 2
AUG = {'crop_size': list(CROP), 'min_scale': -0.1, 'max_scale': 1.0, 'do_flip': True}
LR = (1e-4, 2e-4, 2)                      # cyclical schedule, changing every step


def _write_chairs(root, seed=0):
    from PIL import Image
    from tf_raft_b200.datasets import frame_utils
    rng = np.random.default_rng(seed)
    data = os.path.join(root, 'data')
    os.makedirs(data, exist_ok=True)
    codes = [1] * N_TRAIN + [2] * N_VAL
    rng.shuffle(codes)
    for i in range(len(codes)):
        for t in (1, 2):
            base = rng.integers(0, 256, (H // 8 + 1, W // 8 + 1, 3)).astype(np.uint8)
            Image.fromarray(np.kron(base, np.ones((8, 8, 1), np.uint8))[:H, :W]).save(
                os.path.join(data, f'{i + 1:05d}_img{t}.ppm'))
        frame_utils.write_flow(os.path.join(data, f'{i + 1:05d}_flow.flo'),
                               rng.normal(0, 3, (H, W, 2)).astype(np.float32))
    split = os.path.join(root, 'split.txt')
    np.savetxt(split, np.array(codes), fmt='%d')
    return data, split


@pytest.fixture(scope='module')
def chairs(tmp_path_factory):
    return _write_chairs(str(tmp_path_factory.mktemp('chairs')))


class Batches:
    def __init__(self, ds, batch_size):
        self.ds, self.batch_size = ds, batch_size

    def __iter__(self):
        return iter(self.ds.batches(self.batch_size, workers=2))


class Schedule:
    """The cyclical schedule, recording each (step, value) the optimiser asks for."""

    def __init__(self):
        from tf_raft_b200 import CyclicalLearningRate
        self.f = CyclicalLearningRate(*LR)
        self.calls = []

    def __call__(self, step):
        value = self.f(step)
        self.calls.append((step, value))
        return value


def _model(variant, seed=21, compile=True):
    import tf_raft_b200 as T
    model = (T.RAFT if variant == 'raft' else T.SmallRAFT)(iters=2, iters_pred=2, precision='f16x2')
    model.load_params(weights.init_params(variant, seed, bias_scale=0.05, norm_jitter=0.1))
    sched = Schedule()
    if compile:
        model.compile(optimizer=T.AdamW(weight_decay=1e-4, learning_rate=sched), clip_norm=1.0)
    return model, sched


def _datasets(chairs, seed):
    from tf_raft_b200.datasets import FlyingChairs
    data, split = chairs
    np.random.seed(seed)
    random.seed(seed)
    train = FlyingChairs(AUG, split='training', split_txt=split, root=data)
    train.shuffle()
    return train, FlyingChairs(split='validation', split_txt=split, root=data)


def _close(a, b, atol, rtol=0.0):
    err = float((a.double() - b.double()).abs().max())
    return err, err <= atol + rtol * float(b.double().abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_fit_matches_a_hand_loop_and_checkpoints_the_best_epoch(chairs, tmp_path, variant):
    """fit over batches(..., repeat=True) with validation and two ModelCheckpoints (min and max of val_epe), against
    the same seeds driven by hand: the same batches bit for bit (5 items, 6 batches of 2: the stream wraps inside a
    batch), the schedule's value at steps 0..5 exactly, and end states within the stated tolerance.  Each saved file
    loads into the parameters and moving statistics the model had at the end of that epoch, bit for bit."""
    from tf_raft_b200 import CyclicalLearningRate, ModelCheckpoint, load_tf_checkpoint
    from tf_raft_b200.fit import Callback

    class Snapshot(Callback):
        def __init__(self):
            super().__init__()
            self.states = []

        def on_epoch_end(self, epoch, logs=None):
            self.states.append({k: v.detach().cpu().numpy().copy() for k, v in self.model.state_dict().items()})

    model, sched = _model(variant)
    train, val = _datasets(chairs, 5)
    fed = []
    step = model.train_step

    def recording_step(batch):
        fed.append(tuple(t.clone() for t in batch))
        return step(batch)

    model.train_step = recording_step
    ckpt = {mode: ModelCheckpoint(str(tmp_path / mode / 'model-{epoch}'), monitor='val_epe', mode=mode,
                                  save_best_only=True, save_weights_only=True) for mode in ('min', 'max')}
    snap = Snapshot()
    hist = model.fit(train.batches(BATCH, workers=2, repeat=True), epochs=EPOCHS, steps_per_epoch=STEPS,
                     validation_data=Batches(val, 1), validation_steps=N_VAL,
                     callbacks=[ckpt['min'], ckpt['max'], snap], verbose=0)
    assert len(fed) == EPOCHS * STEPS and model.optimizer.iterations == EPOCHS * STEPS
    ref = CyclicalLearningRate(*LR)
    assert sched.calls == [(s, ref(s)) for s in range(EPOCHS * STEPS)]
    assert hist.history['val_loss'] == [0.0] * EPOCHS

    hand, _ = _model(variant)
    train2, val2 = _datasets(chairs, 5)
    stream = train2.batches(BATCH, workers=2, repeat=True)
    logs = []
    for epoch in range(EPOCHS):
        hand.reset_metrics()
        for s in range(STEPS):
            batch = next(stream)
            for a, b in zip(batch, fed[epoch * STEPS + s]):
                assert a.dtype == b.dtype and torch.equal(a, b), f'epoch {epoch} step {s}: batches differ'
            out = dict(hand.train_step(batch))
        hand.reset_metrics()
        for vb in val2.batches(1, workers=2):
            vout = hand.test_step(vb[:4])
        out.update(('val_' + k, v) for k, v in vout.items())
        logs.append(out)

    # Tolerance: Adam moves an entry by about lr per step whatever the gradient's size, so where a gradient is
    # decided by rounding (the atomicAdd order) the two runs may part by up to that much per step.
    a, b = model._trainer, hand._trainer
    err_p, ok = _close(a.flat.p, b.flat.p, atol=2 * EPOCHS * STEPS * LR[1])
    assert ok, f'parameters differ by {err_p}'
    for name in ('m', 'v'):
        err, ok = _close(getattr(a.flat, name), getattr(b.flat, name), atol=0.0, rtol=5e-2)
        assert ok, f'{name} differs by {err}'
    for k, v in a.moving.items():
        err, ok = _close(v, b.moving[k], atol=0.0, rtol=1e-2)
        assert ok, f'{k} differs by {err}'
    for epoch in range(EPOCHS):
        for k, v in logs[epoch].items():
            assert hist.history[k][epoch] == pytest.approx(v, rel=5e-2, abs=1e-6), (epoch, k)
    print(f'{variant}: fit vs hand loop: parameters {err_p:.2e}, val_epe {hist.history["val_epe"]}')

    epe = hist.history['val_epe']
    for mode, better in (('min', np.less), ('max', np.greater)):
        best, want = np.inf if mode == 'min' else -np.inf, []
        for epoch, e in enumerate(epe):
            if better(e, best):
                best = e
                want.append(epoch + 1)
        got = sorted(int(p.split('-')[-1][:-len('.index')]) for p in glob.glob(str(tmp_path / mode / 'model-*.index')))
        assert got == want, (mode, epe)
        for e in got:
            params = load_tf_checkpoint(str(tmp_path / mode / f'model-{e}'), expect=model.state_dict())
            assert sorted(params) == sorted(snap.states[e - 1])
            for k, v in snap.states[e - 1].items():
                assert params[k].dtype == v.dtype and np.array_equal(params[k], v), (mode, e, k)


def _fixed_batch(seed):
    import cases
    rng = np.random.default_rng(seed)
    im1, im2 = (torch.from_numpy(a).cuda() for a in cases.images(2, 64, 96, 3, 4))
    flow = torch.from_numpy((rng.standard_normal((2, 64, 96, 2)) * 5).astype(np.float32)).cuda()
    valid = torch.from_numpy(rng.uniform(size=(2, 64, 96)) > 0.1).cuda()
    return im1, im2, flow, valid


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_save_weights_then_load_weights_resumes(tmp_path, variant):
    """After 2 steps, save_weights; load_weights into a fresh compiled model (and, in the other order, into a model
    compiled afterwards) gives byte-equal flat parameters, moments, moving statistics and iterations.  Step 3 on the
    same batch then agrees with the original model's within one Adam step (atomicAdd order, see above)."""
    from tf_raft_b200 import checkpoint as ck
    data = _fixed_batch(9)
    model, _ = _model(variant)
    for _ in range(2):
        model.train_step(data)
    prefix = str(tmp_path / 'ckpt' / 'model')
    model.save_weights(prefix)
    raw = ck.read_tf_checkpoint(prefix)
    assert raw[ck.OPTIMIZER_ITER_KEY].dtype == np.int64 and int(raw[ck.OPTIMIZER_ITER_KEY]) == 2
    assert ck.optimizer_slot_key('fnet.conv1.kernel', 'v') in raw

    fresh, _ = _model(variant, seed=99)                   # compiled, other initial values
    fresh.load_weights(prefix)
    later, _ = _model(variant, seed=98, compile=False)
    later.load_weights(prefix)                            # not compiled yet: the optimiser state waits
    assert later._trainer is None
    import tf_raft_b200 as T
    later.compile(optimizer=T.AdamW(weight_decay=1e-4, learning_rate=Schedule()), clip_norm=1.0)
    a = model._trainer
    for other in (fresh, later):
        b = other._trainer
        assert other.optimizer.iterations == 2
        for name in ('p', 'm', 'v'):
            assert torch.equal(getattr(a.flat, name), getattr(b.flat, name)), name
        assert all(torch.equal(v, b.moving[k]) for k, v in a.moving.items())
    model.reset_metrics()
    fresh.reset_metrics()
    out_a = model.train_step(data)
    out_b = fresh.train_step(data)
    assert fresh.optimizer.iterations == 3
    err, ok = _close(fresh._trainer.flat.p, a.flat.p, atol=2 * LR[1])
    assert ok, f'step 3 parameters differ by {err}'
    assert out_b['loss'] == pytest.approx(out_a['loss'], rel=1e-4)
    # weights alone (no optimiser state in the file): moments start at zero and iterations stay
    only = str(tmp_path / 'weights' / 'model')
    ck.write_tf_checkpoint(only, {k: v for k, v in raw.items() if '.OPTIMIZER_SLOT' not in k and k != ck.OPTIMIZER_ITER_KEY})
    plain, _ = _model(variant, seed=97)
    plain.load_weights(only)
    assert plain._trainer is None and plain.optimizer.iterations == 0
    loaded = plain.state_dict()
    saved = ck.load_tf_checkpoint(prefix)
    assert all(np.array_equal(loaded[k].cpu().numpy(), v) for k, v in saved.items())


@pytest.mark.gpu
def test_train_script_runs_and_resumes(chairs, tmp_path):
    """scripts/train.py chairs for one epoch, then again resumed from the first run's checkpoint."""
    yaml = pytest.importorskip('yaml', reason='scripts/train.py reads YAML configs and needs PyYAML')
    from test_fit import read_events
    from tf_raft_b200 import checkpoint as ck
    data, split = chairs
    config = {'data': {'root': data, 'split_txt': split}, 'augment': AUG,
              'model': {'iters': 2, 'iters_pred': 2, 'resume': 0},
              'train': {'epochs': 1, 'batch_size': BATCH, 'learning_rate': 4e-4, 'weight_decay': 1e-4, 'clip_norm': 1},
              'visualize': {'num_visualize': 1, 'choose_random': True}, 'logdir': str(tmp_path / 'logs1')}
    steps = N_TRAIN // BATCH
    runs = []
    for run in range(2):
        cfg = str(tmp_path / f'run{run}.yml')
        with open(cfg, 'w') as f:
            yaml.dump(config, f)
        proc = subprocess.run([sys.executable, os.path.join(ROOT, 'scripts', 'train.py'), 'chairs', cfg, '--seed', '3',
                               '--workers', '2'], capture_output=True, text=True, timeout=1200)
        assert proc.returncode == 0, proc.stdout[-3000:] + proc.stderr[-3000:]
        (logdir,) = glob.glob(os.path.join(config['logdir'], '*'))
        runs.append((logdir, proc.stdout))
        assert os.path.exists(os.path.join(logdir, 'config.yml'))
        for sub in ('train', 'validation'):
            (events,) = glob.glob(os.path.join(logdir, 'history', sub, 'events.out.tfevents.*'))
            tags = {tag for *_, values in read_events(events) for tag, _ in values}
            assert {'epoch_epe', 'epoch_loss'} <= tags
        from PIL import Image
        (png,) = glob.glob(os.path.join(logdir, 'predicted_flows', 'epoch001_*.png'))
        assert Image.open(png).size == (W, 3 * H)
        saved = ck.read_tf_checkpoint(os.path.join(logdir, 'checkpoints', 'model'))
        assert int(saved[ck.OPTIMIZER_ITER_KEY]) == (run + 1) * steps
        config = dict(config, model=dict(config['model'], resume=os.path.join(logdir, 'checkpoints', 'model')),
                      logdir=str(tmp_path / 'logs2'))
    assert f'done (iteration {steps})' in runs[1][1]
