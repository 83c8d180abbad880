"""Train RAFT on FlyingChairs or MPI Sintel with the reference's YAML configs (train_chairs.py, train_sintel.py).

    python scripts/train.py chairs configs/train_chairs.yml [--small] [--seed S] [--workers N]
    python scripts/train.py sintel configs/train_sintel.yml
    python scripts/train.py chairs configs/train_chairs.yml --self-supervised

The config keys are the reference's: data.root (and data.split_txt for chairs), augment.* (the augmentor's
arguments), model.iters / iters_pred / resume, train.epochs / batch_size / learning_rate / weight_decay / clip_norm,
visualize.num_visualize / choose_random, logdir.  A missing key stops the script with its name.

As in the reference: the shuffled training set with steps_per_epoch = len // batch_size over an endless item stream
(`FlowDataset.batches(..., repeat=True)` in the role of tf.data), validation after every epoch at batch 1 (Chairs: the
validation split at its native 384x512; Sintel: the first 10 % of a separately shuffled clean training list,
crop-or-padded to 448x1024), `CyclicalLearningRate(lr, 2 lr, 1000, first_cycle_scaler, 'cycle')` under
`AdamW(weight_decay, schedule)`, and the TensorBoard, VisFlowCallback and ModelCheckpoint(monitor='val_epe',
save_best_only=True) callbacks writing to <logdir>/<timestamp>/{history, predicted_flows, checkpoints/model}, with the
config saved beside them as config.yml.  The timestamp has seconds (the reference's has minutes), so that two runs
started in the same minute do not share a directory.  `model.resume` names a checkpoint prefix written by a previous
run; its weights, Adam moments and step count are restored, so the learning-rate schedule continues.

`--self-supervised` compiles with `UnsupervisedLoss()` (DESIGN.md section 9.1): the training batches' ground truth is not
used by the loss (the epe metrics of the forward prediction are still logged); the config, datasets, validation (val_epe
against ground truth) and callbacks are the same.
"""
import argparse
import os
import random
import sys
from datetime import datetime

import numpy as np

try:
    import yaml
except ImportError:                                    # pragma: no cover - depends on the environment
    sys.exit('scripts/train.py reads YAML configs and needs PyYAML (pip install pyyaml)')

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), '..')))

import tf_raft_b200 as T  # noqa: E402
from tf_raft_b200 import datasets as D  # noqa: E402

VAL_SIZE = {'chairs': None, 'sintel': (448, 1024)}      # validation crop-or-pad target (None: native size)


class Batches:
    """A re-iterable `dataset.batches(...)`: `fit` iterates the validation set afresh every epoch."""

    def __init__(self, dataset, batch_size, **kwargs):
        self.dataset, self.batch_size, self.kwargs = dataset, batch_size, kwargs

    def __iter__(self):
        return iter(self.dataset.batches(self.batch_size, **self.kwargs))


def need(config, path):
    node = config
    for i, key in enumerate(path.split('.')):
        if not isinstance(node, dict) or key not in node:
            sys.exit(f'config: missing key {".".join(path.split(".")[:i + 1])!r}')
        node = node[key]
    return node


def train(name, config, logdir, small=False, workers=4, self_supervised=False, train_precision='fp32'):
    root = need(config, 'data.root')
    aug_params = need(config, 'augment')
    iters, iters_pred, resume = (need(config, 'model.' + k) for k in ('iters', 'iters_pred', 'resume'))
    epochs, batch_size, learning_rate, weight_decay, clip_norm = (
        need(config, 'train.' + k) for k in ('epochs', 'batch_size', 'learning_rate', 'weight_decay', 'clip_norm'))
    num_visualize, choose_random = (need(config, 'visualize.' + k) for k in ('num_visualize', 'choose_random'))

    if name == 'chairs':
        split_txt = need(config, 'data.split_txt')
        ds_train = D.FlyingChairs(aug_params, split='training', split_txt=split_txt, root=root)
        ds_train.shuffle()
        ds_val = D.FlyingChairs(split='validation', split_txt=split_txt, root=root)
        ds_vis = D.FlyingChairs(split='validation', split_txt=split_txt, root=root)
    else:
        ds_train = D.MpiSintel(aug_params, split='training', root=root, dstype='clean')
        ds_train.shuffle()
        ds_val = D.MpiSintel(split='training', root=root, dstype='clean')
        ds_val.shuffle()
        val_size = int(0.1 * len(ds_train))
        ds_val.image_list = ds_val.image_list[:val_size]
        ds_val.flow_list = ds_val.flow_list[:val_size]
        ds_vis = D.MpiSintel(split='training', root=root, dstype='clean')
        ds_vis.shuffle()
    train_size, val_size = len(ds_train), len(ds_val)
    print(f'Found {train_size} samples for training')
    print(f'Found {val_size} samples for validation')

    scheduler = T.CyclicalLearningRate(initial_learning_rate=learning_rate, maximal_learning_rate=2 * learning_rate,
                                       step_size=1000, scale_fn=T.first_cycle_scaler, scale_mode='cycle')
    optimizer = T.AdamW(weight_decay=weight_decay, learning_rate=scheduler)
    raft = (T.SmallRAFT if small else T.RAFT)(drop_rate=0, iters=iters, iters_pred=iters_pred)
    loss = T.UnsupervisedLoss() if self_supervised else T.sequence_loss
    raft.compile(optimizer=optimizer, clip_norm=clip_norm, loss=loss, epe=T.end_point_error,
                 train_precision=train_precision)
    if resume:
        print(f'Restoring pretrained weights from {resume} ...', end=' ')
        raft.load_weights(resume)
        print(f'done (iteration {optimizer.iterations})', flush=True)

    callbacks = [
        T.TensorBoard(log_dir=os.path.join(logdir, 'history')),
        T.VisFlowCallback(ds_vis, num_visualize=num_visualize, choose_random=choose_random,
                          logdir=os.path.join(logdir, 'predicted_flows')),
        T.ModelCheckpoint(filepath=os.path.join(logdir, 'checkpoints', 'model'), save_weights_only=True,
                          monitor='val_epe', mode='min', save_best_only=True),
    ]
    return raft.fit(ds_train.batches(batch_size, workers=workers, repeat=True), epochs=epochs, callbacks=callbacks,
                    steps_per_epoch=train_size // batch_size,
                    validation_data=Batches(ds_val, 1, target_size=VAL_SIZE[name], workers=workers),
                    validation_steps=val_size)


def main():
    parser = argparse.ArgumentParser(description='Train RAFT with a tf-raft config')
    parser.add_argument('dataset', choices=('chairs', 'sintel'))
    parser.add_argument('config', help='YAML config in the reference\'s layout')
    parser.add_argument('--small', action='store_true', help='SmallRAFT instead of RAFT')
    parser.add_argument('--seed', type=int, default=None, help='seed np.random and random before the first shuffle')
    parser.add_argument('--workers', type=int, default=4, help='loader threads')
    parser.add_argument('--train-precision', choices=('fp32', 'f16x2'), default='fp32',
                        help="convolutions of the step: IEEE-fp32 library (fp32) or tensor-core hi/lo (f16x2)")
    parser.add_argument('--self-supervised', action='store_true',
                        help='train with UnsupervisedLoss (census + smoothness, both directions) instead of ground truth')
    args = parser.parse_args()

    with open(args.config) as f:
        config = yaml.load(f, Loader=yaml.SafeLoader)
    logdir = os.path.join(need(config, 'logdir'), datetime.now().strftime('%Y-%m-%dT%H-%M-%S'))
    os.makedirs(logdir, exist_ok=True)
    with open(os.path.join(logdir, 'config.yml'), 'w') as f:
        f.write(yaml.dump(config, default_flow_style=False))
    print('------------ Config ---------------')
    print(yaml.dump(config))
    print('-----------------------------------')
    print(f'logdir: {logdir}', flush=True)
    if args.seed is not None:
        np.random.seed(args.seed)
        random.seed(args.seed)
    train(args.dataset, config, logdir, small=args.small, workers=args.workers, self_supervised=args.self_supervised,
          train_precision=args.train_precision)


if __name__ == '__main__':
    main()
