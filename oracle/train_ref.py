"""Float64 restatement of the optimiser state of the training step (test infrastructure).

What tf_raft/model.py:126-144 and train_chairs.py:79-98 do to the variables after the gradient is known, written out in
plain float64 NumPy so that every CUDA kernel and every piece of host glue of the training step has a truth to be held to:

* `clip_scale`: tf.clip_by_global_norm (tensorflow/python/ops/clip_ops.py) -- every gradient is multiplied by
  `clip_norm / max(global_norm, clip_norm)`, global_norm = sqrt(sum of g^2 over all variables).
* `AdamW`: tfa.optimizers.AdamW = DecoupledWeightDecayExtension over Keras Adam (non-amsgrad), as Keras applies it:
  the decay `var -= wd * var` first (tfa's `_decay_weights_op`, NOT scaled by the learning rate), then Keras Adam
  (`_resource_apply_dense` -> ResourceApplyAdam): m = b1 m + (1-b1) g, v = b2 v + (1-b2) g^2,
  var -= lr_t m / (sqrt(v) + eps), lr_t = lr(iterations) sqrt(1 - b2^t) / (1 - b1^t), t = iterations + 1.  A learning-rate
  schedule is called with `iterations` before the increment (OptimizerV2._decayed_lr).
* `cyclical_lr`: tfa.optimizers.CyclicalLearningRate (scale_mode 'cycle' or 'iterations').
* `bn_moving_update`: keras BatchNormalization on 4-D NHWC input with axis=-1 takes the fused path
  (normalization.py `_fused_batch_norm`); FusedBatchNormV3 in training mode updates the moving variance with the batch
  variance times n / (n - 1) ("rest_size_adjust"; cuDNN does the same), and Keras leaves that correction in because
  `_bessels_correction_test_only` is true outside its legacy tests.  The normalisation itself uses the biased variance.
  moving = momentum * moving + (1 - momentum) * batch statistic, momentum 0.99; n is the number of values per channel
  the statistics were taken over -- under data parallelism with synchronised statistics, the global count.

Restated from the TensorFlow 2.3 / TensorFlow Addons 0.11 sources; not checked against a TensorFlow run.
"""
import math

import numpy as np

F64 = np.float64


def global_sumsq(grads):
    """sum of g^2 over every array of `grads` (a dict or a sequence), in float64."""
    vals = grads.values() if isinstance(grads, dict) else grads
    return float(sum(np.square(np.asarray(g, dtype=F64)).sum() for g in vals))


def clip_scale(sumsq, clip_norm):
    """tf.clip_by_global_norm's factor for a gradient whose squared global norm is `sumsq`; None or 0 disables the clip."""
    if not clip_norm:
        return 1.0
    return float(clip_norm) / max(math.sqrt(sumsq), float(clip_norm))


def cyclical_lr(step, initial, maximal, step_size, scale_fn, scale_mode='cycle'):
    """tfa CyclicalLearningRate.__call__(step)."""
    cycle = math.floor(1 + step / (2 * step_size))
    x = abs(step / step_size - 2 * cycle + 1)
    mode_step = cycle if scale_mode == 'cycle' else step
    return initial + (maximal - initial) * max(0.0, 1 - x) * scale_fn(mode_step)


class AdamW:
    """tfa AdamW state in float64: per-variable m and v, the iteration count, and the update of one apply_gradients."""

    def __init__(self, weight_decay, learning_rate, beta_1=0.9, beta_2=0.999, epsilon=1e-7):
        self.weight_decay, self.learning_rate = float(weight_decay), learning_rate
        self.beta_1, self.beta_2, self.epsilon = float(beta_1), float(beta_2), float(epsilon)
        self.iterations = 0
        self.m, self.v = {}, {}

    def lr(self):
        """the learning rate of the NEXT step: a schedule is evaluated at `iterations` (before the increment)."""
        lr = self.learning_rate
        return float(lr(self.iterations)) if callable(lr) else float(lr)

    def lr_t(self):
        """the bias-corrected step size of the next step, t = iterations + 1."""
        t = self.iterations + 1
        return self.lr() * math.sqrt(1 - self.beta_2 ** t) / (1 - self.beta_1 ** t)

    def apply(self, params, grads, clip_norm=None):
        """clip_by_global_norm + apply_gradients on float64 copies: returns the new {name: value}; m, v and iterations
        advance.  `grads` are the raw (unclipped) gradients."""
        scale = clip_scale(global_sumsq(grads), clip_norm)
        lr_t = self.lr_t()
        b1, b2, eps, wd = self.beta_1, self.beta_2, self.epsilon, self.weight_decay
        out = {}
        for k, g in grads.items():
            g = np.asarray(g, dtype=F64) * scale
            w = np.asarray(params[k], dtype=F64)
            w = w - wd * w
            m = b1 * self.m.get(k, 0.0) + (1 - b1) * g
            v = b2 * self.v.get(k, 0.0) + (1 - b2) * g * g
            self.m[k], self.v[k] = m, v
            out[k] = w - lr_t * m / (np.sqrt(v) + eps)
        self.iterations += 1
        return out


def bn_moving_update(moving, record, momentum=0.99):
    """Advance keras moving statistics by one training-mode forward.  `moving` maps '<layer>.moving_mean' /
    '<layer>.moving_variance' to arrays; `record` maps '<layer>' to (batch mean, biased batch variance, count) as
    `oracle.raft_torch.Ops(..., bn_record=...)` returns them.  Returns new float64 arrays for the recorded layers."""
    out = {}
    for name, (mean, var, n) in record.items():
        mean = np.asarray(mean, dtype=F64)
        var = np.asarray(var, dtype=F64) * (n / (n - 1) if n > 1 else 1.0)
        mm = np.asarray(moving[name + '.moving_mean'], dtype=F64)
        mv = np.asarray(moving[name + '.moving_variance'], dtype=F64)
        out[name + '.moving_mean'] = momentum * mm + (1 - momentum) * mean
        out[name + '.moving_variance'] = momentum * mv + (1 - momentum) * var
    return out
