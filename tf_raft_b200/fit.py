"""`RAFT.fit`: Keras's (TensorFlow 2.3) `Model.fit` loop as the reference's training scripts use it
(train_chairs.py:122-129, train_sintel.py:126-133), as a function of the model so that any object with `train_step`,
`test_step` and `reset_metrics` can be driven by it.

Kept from Keras:
* `x` with `steps_per_epoch`: ONE iterator serves every epoch, epoch e takes the next `steps_per_epoch` batches (the
  reference's generator never ends; here `FlowDataset.batches(..., repeat=True)`).  Without it every epoch iterates `x`
  afresh until it is exhausted.  An iterator that runs dry before `steps_per_epoch` ends training after that epoch,
  with a warning, as Keras does.
* `model.reset_metrics()` at the start of every epoch and again before validation (train and test steps share the
  model's `flow_metrics`).  The epoch's training logs are those the epoch's last `train_step` returned.
* Validation iterates `validation_data` afresh every epoch, up to `validation_steps` batches, through `test_step`;
  its logs join the epoch's as `val_<name>`.  `test_step` never updates `loss`, so `val_loss` is the mean over nothing,
  0.0, as in the reference.
* Callbacks are called in list order, then `History`, which records every epoch's logs; `fit` returns it and sets
  `model.history`.
Not kept: `initial_epoch`, `class_weight`, progress bars (verbose=1 prints one line per epoch), `on_*_batch_begin`.
"""
import copy
import itertools
import time
import warnings


class Callback:
    """The subset of `tf.keras.callbacks.Callback` that `fit` calls."""

    def __init__(self):
        self.model = None

    def set_model(self, model):
        self.model = model

    def on_train_begin(self, logs=None):
        pass

    def on_train_end(self, logs=None):
        pass

    def on_epoch_begin(self, epoch, logs=None):
        pass

    def on_epoch_end(self, epoch, logs=None):
        pass

    def on_train_batch_end(self, step, logs=None):
        pass


class History(Callback):
    """`epoch` is the list of epoch indices, `history[name]` the list of that log's values per epoch."""

    def on_train_begin(self, logs=None):
        self.epoch = []
        self.history = {}

    def on_epoch_end(self, epoch, logs=None):
        self.epoch.append(epoch)
        for k, v in (logs or {}).items():
            self.history.setdefault(k, []).append(v)


def _world_size():
    import torch.distributed as dist
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def fit(model, x, epochs=1, callbacks=None, steps_per_epoch=None, validation_data=None, validation_steps=None,
        verbose=1):
    """Runs `epochs` epochs of `model.train_step` over `x`, an iterable of (image1, image2, flow, valid) batches, with
    validation on `validation_data` (4-tuples, or the evaluation loader's 5-tuples whose `sizes` are ignored) after
    each epoch.  Returns the `History`.  Single process only: under a process group of world size > 1 it raises
    (sharded training is `parallel.shard_batch` plus `train_step`)."""
    if _world_size() > 1:
        raise RuntimeError('fit runs in a single process; shard batches with parallel.shard_batch and call train_step')
    if steps_per_epoch is not None and steps_per_epoch < 1:
        raise ValueError('steps_per_epoch must be >= 1')
    # what is iterated afresh every epoch must be re-iterable (a list, or an object whose __iter__ restarts it), not a
    # generator, which would be empty from the second epoch on
    for name, data, fresh in (('x', x, steps_per_epoch is None), ('validation_data', validation_data, True)):
        if fresh and epochs > 1 and data is not None and iter(data) is data:
            raise ValueError(f'{name} is a one-shot iterator but is iterated afresh every epoch; pass a re-iterable '
                             '(e.g. an object whose __iter__ calls FlowDataset.batches)')
    history = History()
    callbacks = list(callbacks or []) + [history]
    for cb in callbacks:
        cb.set_model(model)
    for cb in callbacks:
        cb.on_train_begin()
    stream = iter(x) if steps_per_epoch is not None else None
    for epoch in range(epochs):
        start = time.perf_counter()
        model.reset_metrics()
        for cb in callbacks:
            cb.on_epoch_begin(epoch)
        batches = stream if stream is not None else iter(x)
        logs, step, exhausted = None, 0, False
        while steps_per_epoch is None or step < steps_per_epoch:
            try:
                batch = next(batches)
            except StopIteration:
                exhausted = steps_per_epoch is not None
                break
            logs = model.train_step(batch)
            for cb in callbacks:
                cb.on_train_batch_end(step, logs)
            step += 1
        if logs is None:
            raise ValueError(f'epoch {epoch + 1}: the training data yielded no batch')
        if exhausted:
            warnings.warn(f'the training data ran out after {step} of {steps_per_epoch} steps of epoch {epoch + 1}; '
                          'training stops after this epoch')
        epoch_logs = dict(logs)
        if validation_data is not None:
            epoch_logs.update(('val_' + k, v) for k, v in _validate(model, validation_data, validation_steps).items())
        for cb in callbacks:
            cb.on_epoch_end(epoch, epoch_logs)
        if verbose:
            items = ' - '.join(f'{k}: {v:.4f}' for k, v in epoch_logs.items())
            print(f'Epoch {epoch + 1}/{epochs} - {step} steps - {time.perf_counter() - start:.1f}s - {items}', flush=True)
        if exhausted:
            break
    for cb in callbacks:
        cb.on_train_end()
    model.history = history
    return history


def _validate(model, data, steps):
    """Keras's `evaluate` inside `fit`: metrics reset, then `test_step` on each batch; the last step's logs."""
    model.reset_metrics()
    logs = {}
    for batch in itertools.islice(data, steps):
        logs = model.test_step(tuple(batch[:4]))
    return copy.copy(logs)
