"""`fit`, `ModelCheckpoint`, the TensorBoard event writer and the checkpoint key inverse, on the CPU with a stub model
(tf_raft_b200/fit.py, tf_raft_b200/train.py, tf_raft_b200/checkpoint.py)."""
import glob
import os
import struct

import numpy as np
import pytest

from oracle import weights
from tf_raft_b200 import checkpoint as ck
from tf_raft_b200.fit import Callback, fit
from tf_raft_b200.train import ModelCheckpoint, TensorBoard


class StubModel:
    """train_step / test_step record their calls in `calls` and return scripted logs."""

    def __init__(self):
        self.calls = []
        self.saved = []
        self.n_train = self.n_test = 0

    def reset_metrics(self):
        self.calls.append(('reset',))

    def train_step(self, batch):
        self.calls.append(('train', batch))
        self.n_train += 1
        return {'loss': float(self.n_train), 'epe': 10.0 * self.n_train}

    def test_step(self, batch):
        self.calls.append(('test', batch))
        self.n_test += 1
        return {'loss': 0.0, 'epe': 100.0 * self.n_test}

    def save_weights(self, path):
        self.saved.append(path)


class Recorder(Callback):
    def __init__(self, name, log):
        super().__init__()
        self.name, self.log = name, log

    def set_model(self, model):
        super().set_model(model)
        self.log.append((self.name, 'set_model'))

    def on_train_begin(self, logs=None):
        self.log.append((self.name, 'train_begin'))

    def on_train_end(self, logs=None):
        self.log.append((self.name, 'train_end'))

    def on_epoch_begin(self, epoch, logs=None):
        self.log.append((self.name, 'epoch_begin', epoch))

    def on_epoch_end(self, epoch, logs=None):
        self.log.append((self.name, 'epoch_end', epoch, dict(logs)))

    def on_train_batch_end(self, step, logs=None):
        self.log.append((self.name, 'batch_end', step, dict(logs)))


def _batch(i):
    return ('im1', 'im2', 'flow', i)


def _trained(model):
    return [c[1][3] for c in model.calls if c[0] == 'train']


def test_steps_per_epoch_continues_one_iterator_across_epochs():
    model = StubModel()
    stream = (_batch(i) for i in range(100))                        # an endless-style generator, read once
    hist = fit(model, stream, epochs=3, steps_per_epoch=4, verbose=0)
    assert _trained(model) == list(range(12))
    assert next(stream) == _batch(12)                                 # nothing read ahead
    assert hist.epoch == [0, 1, 2]
    assert hist.history['loss'] == [4.0, 8.0, 12.0]                   # the last step's logs of each epoch
    assert model.history is hist


def test_without_steps_per_epoch_each_epoch_iterates_afresh():
    model = StubModel()
    data = [_batch(i) for i in range(3)]
    fit(model, data, epochs=2, verbose=0)
    assert _trained(model) == [0, 1, 2, 0, 1, 2]
    with pytest.raises(ValueError, match='one-shot'):
        fit(StubModel(), iter(data), epochs=2, verbose=0)
    with pytest.raises(ValueError, match='no batch'):
        fit(StubModel(), [], epochs=1, verbose=0)


def test_running_dry_stops_after_the_epoch():
    model = StubModel()
    with pytest.warns(UserWarning, match='ran out'):
        hist = fit(model, iter([_batch(i) for i in range(5)]), epochs=4, steps_per_epoch=3, verbose=0)
    assert _trained(model) == [0, 1, 2, 3, 4] and hist.epoch == [0, 1]


def test_resets_validation_and_val_logs():
    model = StubModel()
    val = [(*_batch(100 + i), [(8, 8)]) for i in range(5)]             # the evaluation loader's 5-tuples
    hist = fit(model, [_batch(i) for i in range(100)], epochs=2, steps_per_epoch=2, validation_data=val,
               validation_steps=3, verbose=0)
    kinds = [c[0] if c[0] == 'reset' else (c[0], c[1][3]) for c in model.calls]
    assert kinds == ['reset', ('train', 0), ('train', 1), 'reset', ('test', 100), ('test', 101), ('test', 102),
                     'reset', ('train', 2), ('train', 3), 'reset', ('test', 100), ('test', 101), ('test', 102)]
    assert all(len(c[1]) == 4 for c in model.calls if c[0] == 'test')  # sizes dropped
    # val_loss is 0.0: test_step never updates the loss metric (the reference's quirk)
    assert hist.history == {'loss': [2.0, 4.0], 'epe': [20.0, 40.0], 'val_loss': [0.0, 0.0], 'val_epe': [300.0, 600.0]}


def test_callback_order_and_arguments():
    log = []
    model = StubModel()
    hist = fit(model, [_batch(i) for i in range(10)], epochs=2, steps_per_epoch=2,
               callbacks=[Recorder('a', log), Recorder('b', log)], validation_data=[_batch(50)], verbose=0)
    assert log[:4] == [('a', 'set_model'), ('b', 'set_model'), ('a', 'train_begin'), ('b', 'train_begin')]
    e0 = {'loss': 2.0, 'epe': 20.0, 'val_loss': 0.0, 'val_epe': 100.0}
    assert log[4:12] == [('a', 'epoch_begin', 0), ('b', 'epoch_begin', 0),
                         ('a', 'batch_end', 0, {'loss': 1.0, 'epe': 10.0}), ('b', 'batch_end', 0, {'loss': 1.0, 'epe': 10.0}),
                         ('a', 'batch_end', 1, {'loss': 2.0, 'epe': 20.0}), ('b', 'batch_end', 1, {'loss': 2.0, 'epe': 20.0}),
                         ('a', 'epoch_end', 0, e0), ('b', 'epoch_end', 0, e0)]
    assert log[-2:] == [('a', 'train_end'), ('b', 'train_end')]
    assert len(log) == 22
    assert hist.history['val_epe'] == [100.0, 200.0]


def test_fit_refuses_a_process_group(monkeypatch):
    from tf_raft_b200 import fit as fit_module
    monkeypatch.setattr(fit_module, '_world_size', lambda: 2)
    with pytest.raises(RuntimeError, match='single process'):
        fit(StubModel(), [_batch(0)], verbose=0)


# ---------------------------------------------------------------------------------------------------- ModelCheckpoint
EPES = [5.0, 4.0, 4.0, 6.0, 3.0]


def _drive(cb, logs_seq):
    model = StubModel()
    cb.set_model(model)
    for epoch, logs in enumerate(logs_seq):
        cb.on_epoch_end(epoch, logs)
    return model.saved


@pytest.mark.parametrize('mode,monitor,want', [
    ('min', 'val_epe', [1, 2, 5]),                        # ties (epoch 3) do not count as improvements
    ('auto', 'val_epe', [1, 2, 5]),                       # no 'acc' in the name: min
    ('max', 'val_epe', [1, 4]),
    ('auto', 'val_acc', [1, 4]),                          # 'acc' in the name: max
])
def test_checkpoint_save_best_only(mode, monitor, want):
    cb = ModelCheckpoint('ck/model-{epoch:02d}-{val_loss:.1f}', monitor=monitor, mode=mode, save_best_only=True,
                         save_weights_only=True)
    saved = _drive(cb, [{'loss': 1.0, 'val_loss': 0.0, monitor: e} for e in EPES])
    assert saved == [f'ck/model-{e:02d}-0.0' for e in want]


def test_checkpoint_every_epoch_and_missing_monitor():
    assert _drive(ModelCheckpoint('m{epoch}', save_weights_only=True), [{}, {}]) == ['m1', 'm2']
    cb = ModelCheckpoint('m', monitor='val_epe', save_best_only=True, save_weights_only=True)
    with pytest.warns(UserWarning, match='val_epe available'):
        assert _drive(cb, [{'epe': 1.0}]) == []
    with pytest.raises(ValueError, match='save_weights_only'):
        ModelCheckpoint('m', save_weights_only=False)


# ------------------------------------------------------------------------------------------------ TensorBoard events
def _crc32c(data):
    crc = 0xFFFFFFFF
    for byte in data:
        crc ^= byte
        for _ in range(8):
            crc = (crc >> 1) ^ (0x82F63B78 if crc & 1 else 0)
    return crc ^ 0xFFFFFFFF


def _masked(data):
    crc = _crc32c(data)
    return ((((crc >> 15) | (crc << 17)) & 0xFFFFFFFF) + 0xa282ead8) & 0xFFFFFFFF


def _varint(buf, pos):
    shift = value = 0
    while True:
        b = buf[pos]
        pos += 1
        value |= (b & 0x7F) << shift
        if b < 0x80:
            return value, pos
        shift += 7


def _proto(buf):
    """{field: [values]} of one protobuf message (varint, fixed64, bytes and fixed32 fields)."""
    out, pos = {}, 0
    while pos < len(buf):
        tag, pos = _varint(buf, pos)
        field, wire = tag >> 3, tag & 7
        if wire == 0:
            v, pos = _varint(buf, pos)
        elif wire == 1:
            v, pos = buf[pos:pos + 8], pos + 8
        elif wire == 2:
            n, pos = _varint(buf, pos)
            v, pos = buf[pos:pos + n], pos + n
        elif wire == 5:
            v, pos = buf[pos:pos + 4], pos + 4
        else:
            raise AssertionError(f'wire type {wire}')
        out.setdefault(field, []).append((wire, v))
    return out


def read_events(path):
    """[(wall_time, step, file_version or None, [(tag, value)])] of a TFRecord file, both CRCs checked."""
    raw, pos, events = open(path, 'rb').read(), 0, []
    while pos < len(raw):
        header = raw[pos:pos + 8]
        (n,) = struct.unpack('<Q', header)
        assert struct.unpack('<I', raw[pos + 8:pos + 12])[0] == _masked(header), 'length crc'
        data = raw[pos + 12:pos + 12 + n]
        assert struct.unpack('<I', raw[pos + 12 + n:pos + 16 + n])[0] == _masked(data), 'data crc'
        pos += 16 + n
        ev = _proto(data)
        assert ev[1][0][0] == 1
        wall = struct.unpack('<d', ev[1][0][1])[0]
        step = ev[2][0][1] if 2 in ev else 0
        version = bytes(ev[3][0][1]).decode() if 3 in ev else None
        values = []
        for _, summary in ev.get(5, []):
            for _, value in _proto(summary)[1]:
                v = _proto(value)
                assert v[2][0][0] == 5
                values.append((bytes(v[1][0][1]).decode(), struct.unpack('<f', v[2][0][1])[0]))
        events.append((wall, step, version, values))
    return events


def test_tensorboard_event_files(tmp_path):
    cb = TensorBoard(log_dir=str(tmp_path / 'history'))
    cb.set_model(StubModel())
    cb.on_train_begin()
    logs = [{'loss': 1.5, 'epe': 2.25, 'val_loss': 0.0, 'val_epe': 3.5},
            {'loss': 0.75, 'epe': 1.125, 'val_loss': 0.0, 'val_epe': 1e-3}]
    for epoch, l in enumerate(logs):
        cb.on_epoch_end(epoch, l)
    cb.on_train_end()
    for sub, keys in (('train', ('loss', 'epe')), ('validation', ('val_loss', 'val_epe'))):
        files = glob.glob(str(tmp_path / 'history' / sub / 'events.out.tfevents.*'))
        assert len(files) == 1
        name = os.path.basename(files[0]).split('.')
        assert name[-1] == 'v2' and name[3].isdigit() and len(name[3]) == 10 and name[-3] == str(os.getpid())
        events = read_events(files[0])
        assert events[0][2] == 'brain.Event:2' and events[0][3] == []
        got = [(step, values) for _, step, _, values in events[1:]]
        want = [(epoch, [('epoch_' + k.replace('val_', ''), np.float32(l[k]))]) for epoch, l in enumerate(logs)
                for k in keys]
        assert got == want
        assert all(abs(w - events[0][0]) < 60 for w, *_ in events)


# ------------------------------------------------------------------------------------------------ checkpoint keys
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_inverse_key_mapping_round_trips(tmp_path, variant):
    params = weights.init_params(variant, 7)
    keys = {k: ck.param_to_tf_key(k) for k in params}
    assert len(set(keys.values())) == len(params)
    for k, key in keys.items():
        assert ck.tf_key_to_param(key) == k
    assert ck.param_to_tf_key('fnet.layer2.0.downsample.1.gamma') == \
        'fnet/layer2/layer_with_weights-0/downsample/layer_with_weights-1/gamma/.ATTRIBUTES/VARIABLE_VALUE'
    if variant == 'raft':
        assert ck.param_to_tf_key('update_block.mask.2.kernel') == \
            'update_block/mask/layer_with_weights-1/kernel/.ATTRIBUTES/VARIABLE_VALUE'
        assert ck.param_to_tf_key('cnet.norm1.moving_mean') == 'cnet/norm1/moving_mean/.ATTRIBUTES/VARIABLE_VALUE'
    tensors = {keys[k]: np.asarray(v) for k, v in params.items()}
    tensors[ck.OPTIMIZER_ITER_KEY] = np.array(12, dtype=np.int64)
    for k, v in params.items():
        for slot in ('m', 'v'):
            tensors[ck.optimizer_slot_key(k, slot)] = np.full(np.shape(v), 0.5, np.float32)
    assert ck.optimizer_slot_key('fnet.conv1.kernel', 'm') == \
        'fnet/conv1/kernel/.OPTIMIZER_SLOT/optimizer/m/.ATTRIBUTES/VARIABLE_VALUE'
    prefix = str(tmp_path / 'model')
    ck.write_tf_checkpoint(prefix, tensors)
    got = ck.load_tf_checkpoint(prefix, expect=params)
    assert set(got) == set(params)
    for k, v in params.items():
        assert got[k].dtype == np.asarray(v).dtype and np.array_equal(got[k], np.asarray(v)), k
    raw = ck.read_tf_checkpoint(prefix)
    assert raw[ck.OPTIMIZER_ITER_KEY].dtype == np.int64 and int(raw[ck.OPTIMIZER_ITER_KEY]) == 12
