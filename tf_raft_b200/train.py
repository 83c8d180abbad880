"""Training step of RAFT / SmallRAFT -- host-side mirror of tf_raft/model.py:126-144 (GradientTape over the forward with
`training=True`, `clip_by_global_norm`, `apply_gradients`), the optimiser set-up of train_chairs.py:79-98
(tfa AdamW + CyclicalLearningRate) and the scale function of tf_raft/training.py:10-15.

What runs where (DESIGN.md "Training"):
* correlation pyramid forward: the wgmma kernels of the inference path (CorrBlock); backward: two fp32 GEMMs per level;
* pyramid lookup forward AND backward (d/d coords -- the reference does not detach coords1, model.py:102 -- and the
  scatter of d/d pyramid): hand-written CUDA (raft_b200_corr_lookup / raft_b200_corr_lookup_backward);
* global-norm clipping + AdamW on ONE flat fp32 parameter / gradient / moment buffer: hand-written CUDA
  (raft_b200_sumsq, raft_b200_adamw_step);
* data parallelism: one flat all-reduce (NCCL over NVLink) of the 21 MB gradient buffer per step, issued before the
  clipping (global norm of the reduced gradient, as a single-device step on the global batch would compute), and the
  per-channel batch statistics of the context encoder's BatchNorm layers all-reduced in forward and backward (SyncBN:
  the single-device reference normalises over the global batch);
* convolutions, norms, gates, convex upsampling and the loss in the backward-capable form: IEEE-fp32 PyTorch CUDA kernels
  through torch.autograd, with cuDNN switched off for the step (see Trainer.step) -- library code, stated as such;
* with `compile(train_precision='f16x2')`, every stride-1 convolution with cin >= 64 and 'same' (or 1x1 'valid') padding
  runs forward, input gradient and weight gradient on hand-written tensor-core kernels instead (_ConvTC); the rest of
  the list above is unchanged.
"""
import ctypes
import math
import os
import socket
import struct
import time
import warnings

import numpy as np
import torch
import torch.distributed as dist
import torch.nn.functional as F

from . import _lib
from .checkpoint import _field, _mask, _put_varint, crc32c
from .datasets.flow_viz import flow_to_image
from .datasets.frame_utils import write_png
from .fit import Callback
from .layers.corr import CorrBlock
from .layers._params import _same_pads
from .layers.extractor import force_ieee_fp32
from .losses import UnsupervisedLoss, end_point_error, sequence_loss
from .preprocess import resize_with_crop_or_pad

force_ieee_fp32()


# ------------------------------------------------------------------------------------------------ schedules / optimiser
def first_cycle_scaler(cycle):
    """tf_raft/training.py:10-15: 1 during the first cycle, 0 afterwards (min_lr -> max_lr -> min_lr -> const)."""
    return 1.0 if cycle == 1 else 0.0


def inverse_scaler(cycle):
    """tf_raft/training.py:18-23."""
    return 1.0 / cycle


class VisFlowCallback(Callback):
    """tf_raft/training.py:26-88: at the end of each epoch, writes the model's prediction on a few dataset items as
    PNGs: image1, image2 and the flow colour wheel stacked vertically, `epoch{e+1:03d}_{i+1:03d}.png` in `logdir`.

    dataset: a sequence whose items begin with (image1, image2), each H x W x 3 in 0..255 (NumPy arrays or tensors);
    an item with a batch axis raises ValueError.  Item ids are range(num_visualize), or with choose_random
    `np.random.choice(len(dataset), size=num_visualize, replace=False)`, the reference's call on the global NumPy
    generator, so a seeded run picks the reference's ids.  Each pair is crop-or-padded to target_size
    (`resize_with_crop_or_pad`), the model's final prediction (`last_only=True`) is cropped back to H x W and coloured
    on the GPU by `flow_to_image`.  The images are written as uint8: values are clipped to 0..255 and truncated."""

    def __init__(self, dataset, target_size=(448, 1024), num_visualize=1, choose_random=False,
                 logdir='predicted_flows'):
        self.dataset = dataset
        self.target_size = tuple(target_size)
        self.num_visualize = num_visualize
        self.choose_random = choose_random
        self.logdir = logdir
        self.model = None
        os.makedirs(logdir, exist_ok=True)

    @staticmethod
    def _uint8(image):
        image = image.detach().cpu().numpy() if isinstance(image, torch.Tensor) else np.asarray(image)
        return image if image.dtype == np.uint8 else np.clip(image, 0, 255).astype(np.uint8)

    def on_epoch_end(self, epoch, logs=None):
        if self.choose_random:
            vis_ids = np.random.choice(len(self.dataset), size=self.num_visualize, replace=False)
        else:
            vis_ids = range(self.num_visualize)
        device = self.model.device
        for i in vis_ids:
            image1, image2, *_ = self.dataset[i]
            if len(image1.shape) > 3:
                raise ValueError('target dataset must not be batched')
            h, w, _ = image1.shape
            pair = [resize_with_crop_or_pad(torch.as_tensor(np.asarray(im) if not isinstance(im, torch.Tensor) else im,
                                                            dtype=torch.float32, device=device), *self.target_size)[None]
                    for im in (image1, image2)]
            flow = self.model(pair, training=False, last_only=True)[-1][0]
            flow_img = flow_to_image(resize_with_crop_or_pad(flow, h, w)).cpu().numpy()
            contents = np.concatenate([self._uint8(image1), self._uint8(image2), flow_img], axis=0)
            write_png(os.path.join(self.logdir, f'epoch{epoch + 1:03d}_{i + 1:03d}.png'), contents)


class ModelCheckpoint(Callback):
    """tf.keras.callbacks.ModelCheckpoint (TensorFlow 2.3) with save_freq='epoch', as the reference's scripts use it
    (train_chairs.py:113-119): at the end of each epoch, `model.save_weights(filepath.format(epoch=epoch + 1, **logs))`.

    save_best_only: save only when `logs[monitor]` strictly improves on the best value so far, which starts at +inf
    (mode 'min') or -inf ('max'); 'auto' is 'max' when 'acc' is in the monitor's name, else 'min'.  A missing monitor
    warns and does not save.  Only `save_weights_only=True` is supported (no SavedModel)."""

    def __init__(self, filepath, monitor='val_loss', verbose=0, save_best_only=False, save_weights_only=False,
                 mode='auto'):
        super().__init__()
        if not save_weights_only:
            raise ValueError('ModelCheckpoint saves weights only (save_weights_only=True); there is no SavedModel')
        if mode not in ('auto', 'min', 'max'):
            warnings.warn(f'ModelCheckpoint mode {mode} is unknown, fallback to auto mode.')
            mode = 'auto'
        if mode == 'auto':
            mode = 'max' if 'acc' in monitor else 'min'
        self.filepath = os.fspath(filepath)
        self.monitor = monitor
        self.verbose = verbose
        self.save_best_only = save_best_only
        self.monitor_op = np.less if mode == 'min' else np.greater
        self.best = np.inf if mode == 'min' else -np.inf

    def on_epoch_end(self, epoch, logs=None):
        logs = logs or {}
        filepath = self.filepath.format(epoch=epoch + 1, **logs)
        if self.save_best_only:
            current = logs.get(self.monitor)
            if current is None:
                warnings.warn(f'Can save best model only with {self.monitor} available, skipping.')
                return
            if not self.monitor_op(current, self.best):
                if self.verbose:
                    print(f'\nEpoch {epoch + 1:05d}: {self.monitor} did not improve from {self.best:.5f}')
                return
            if self.verbose:
                print(f'\nEpoch {epoch + 1:05d}: {self.monitor} improved from {self.best:.5f} to {current:.5f}, '
                      f'saving model to {filepath}')
            self.best = current
        elif self.verbose:
            print(f'\nEpoch {epoch + 1:05d}: saving model to {filepath}')
        self.model.save_weights(filepath)


class _EventWriter:
    """One TensorBoard event file: TFRecord framing (uint64 length, masked crc32c of the length, the `Event` proto,
    masked crc32c of the proto), first record `file_version: "brain.Event:2"`."""

    _count = 0

    def __init__(self, logdir):
        os.makedirs(logdir, exist_ok=True)
        _EventWriter._count += 1
        name = f'events.out.tfevents.{int(time.time()):010d}.{socket.gethostname()}.{os.getpid()}.{self._count}.v2'
        self.path = os.path.join(logdir, name)
        self.file = open(self.path, 'wb')
        # Event: wall_time = 1 (double), step = 2 (int64), file_version = 3 (string), summary = 5
        self._write(_field(1, 1, struct.pack('<d', time.time())) + _field(3, 2, _bytes(b'brain.Event:2')))

    def _write(self, event):
        length = struct.pack('<Q', len(event))
        self.file.write(length + struct.pack('<I', _mask(crc32c(length))) + event +
                        struct.pack('<I', _mask(crc32c(event))))

    def scalar(self, tag, value, step):
        """Summary{value = 1 {tag = 1, simple_value = 2 (float)}} at `step`."""
        summary_value = _field(1, 2, _bytes(tag.encode('utf-8'))) + _field(2, 5, struct.pack('<f', float(value)))
        self._write(_field(1, 1, struct.pack('<d', time.time())) + _field(2, 0, _put_varint(int(step))) +
                    _field(5, 2, _bytes(_field(1, 2, _bytes(summary_value)))))

    def close(self):
        self.file.close()


def _bytes(payload):
    return _put_varint(len(payload)) + payload


class TensorBoard(Callback):
    """tf.keras.callbacks.TensorBoard (TensorFlow 2.3) with update_freq='epoch', scalars only: at the end of each epoch
    every log `name` becomes the scalar `epoch_<name>` at step = epoch index, the training logs in
    `log_dir/train`, the `val_` logs (prefix stripped) in `log_dir/validation`, one event per scalar.  No graph,
    histograms, images or profiling.  Keras's `tf.summary.scalar` stores the value as a tensor with scalar-plugin
    metadata; this writes the `simple_value` field, which TensorBoard's scalar dashboard reads as well.  These
    semantics come from reading TensorFlow 2.3's Keras sources, not from a TensorFlow run."""

    def __init__(self, log_dir='logs'):
        super().__init__()
        self.log_dir = os.fspath(log_dir)
        self._writers = {}

    def on_epoch_end(self, epoch, logs=None):
        logs = logs or {}
        for name, items in (('train', {k: v for k, v in logs.items() if not k.startswith('val_')}),
                            ('validation', {k[4:]: v for k, v in logs.items() if k.startswith('val_')})):
            if not items:
                continue
            if name not in self._writers:
                self._writers[name] = _EventWriter(os.path.join(self.log_dir, name))
            writer = self._writers[name]
            for k, v in items.items():
                writer.scalar('epoch_' + k, v, epoch)
            writer.file.flush()

    def on_train_end(self, logs=None):
        for writer in self._writers.values():
            writer.close()
        self._writers = {}


class CyclicalLearningRate:
    """tfa.optimizers.CyclicalLearningRate with scale_mode='cycle' (train_chairs.py:79-85)."""

    def __init__(self, initial_learning_rate, maximal_learning_rate, step_size, scale_fn=first_cycle_scaler,
                 scale_mode='cycle'):
        if scale_mode not in ('cycle', 'iterations'):
            raise ValueError(f'unknown scale_mode {scale_mode!r}')
        self.initial_learning_rate = float(initial_learning_rate)
        self.maximal_learning_rate = float(maximal_learning_rate)
        self.step_size = float(step_size)
        self.scale_fn = scale_fn
        self.scale_mode = scale_mode

    def __call__(self, step):
        cycle = math.floor(1 + step / (2 * self.step_size))
        x = abs(step / self.step_size - 2 * cycle + 1)
        mode_step = cycle if self.scale_mode == 'cycle' else step
        return self.initial_learning_rate + (self.maximal_learning_rate - self.initial_learning_rate) * max(0.0, 1 - x) * \
            self.scale_fn(mode_step)


class AdamW:
    """tfa.optimizers.AdamW as configured in train_chairs.py:87-90: Adam (beta 0.9 / 0.999, epsilon 1e-7, no amsgrad) with
    decoupled weight decay `var -= weight_decay * var` (tfa's DecoupledWeightDecayExtension does not multiply by the
    learning rate).  The update itself is one CUDA kernel over a flat buffer (see FlatState.apply)."""

    def __init__(self, weight_decay, learning_rate=1e-3, beta_1=0.9, beta_2=0.999, epsilon=1e-7):
        self.weight_decay = weight_decay
        self.learning_rate = learning_rate
        self.beta_1, self.beta_2, self.epsilon = beta_1, beta_2, epsilon
        self.iterations = 0

    def lr(self):
        lr = self.learning_rate
        return float(lr(self.iterations)) if callable(lr) else float(lr)


# ------------------------------------------------------------------------------------------------ flat parameter state
class FlatState:
    """All trainable variables of a model as views into ONE fp32 buffer (plus gradient and Adam moments of the same
    layout): one all-reduce, one norm reduction, one optimiser launch per step."""

    def __init__(self, params, trainable):
        names = [k for k in params if trainable(k)]
        self.names = names
        device = params[names[0]].device
        sizes = [params[k].numel() for k in names]
        self.offsets = [0]
        for s in sizes:
            self.offsets.append(self.offsets[-1] + (s + 3) // 4 * 4)        # 16-byte aligned slices
        n = self.offsets[-1]
        self.p = torch.zeros(n, dtype=torch.float32, device=device)
        self.g = torch.zeros_like(self.p)
        self.m = torch.zeros_like(self.p)
        self.v = torch.zeros_like(self.p)
        self.views = {}
        for k, o, s in zip(names, self.offsets, sizes):
            view = self.p[o:o + s].view(params[k].shape)
            view.copy_(params[k])
            leaf = view.detach().requires_grad_(True)                          # shares storage with the flat buffer
            leaf.grad = self.g[o:o + s].view(params[k].shape)
            self.views[k] = leaf
        self._norm = torch.zeros(1, dtype=torch.float32, device=device)
        self._part = torch.zeros(1024, dtype=torch.float32, device=device)

    def slot(self, buf):
        """`{name: view}` of a buffer in this layout (self.m, self.v, or a host copy of one), shaped as the variables."""
        return {k: buf[o:o + v.numel()].view(v.shape) for (k, v), o in zip(self.views.items(), self.offsets)}

    def zero_grad(self):
        self.g.zero_()

    def global_norm(self):
        """sqrt(sum g^2) over every trainable variable (tf.linalg.global_norm), on the device."""
        _lib.call('sumsq', self.g.device, _lib.ptr(self.g), self.g.numel(), _lib.ptr(self._part), self._part.numel(),
                  _lib.ptr(self._norm))
        return self._norm                                                    # device scalar: sum of squares

    def apply(self, opt, clip_norm):
        """clip_by_global_norm (model.py:135) + AdamW apply_gradients (:136), one launch; no host synchronisation."""
        sumsq = self.global_norm()
        opt.iterations += 1
        t = opt.iterations
        lr = opt.lr() if not callable(opt.learning_rate) else float(opt.learning_rate(t - 1))
        lr_t = lr * math.sqrt(1 - opt.beta_2 ** t) / (1 - opt.beta_1 ** t)
        _lib.call('adamw_step', self.g.device, _lib.ptr(self.p), _lib.ptr(self.g), _lib.ptr(self.m), _lib.ptr(self.v),
                  self.p.numel(), _lib.ptr(sumsq), float(clip_norm if clip_norm else 0.0), float(lr_t), float(opt.beta_1),
                  float(opt.beta_2), float(opt.epsilon), float(opt.weight_decay))


# ------------------------------------------------------------------------------------------------ autograd pieces
class _Lookup(torch.autograd.Function):
    """CorrBlock.retrieve with gradients to the coordinates and to every pyramid level (hand-written CUDA both ways)."""

    @staticmethod
    def forward(ctx, coords, radius, *pyramid):
        coords = coords.contiguous()
        b, h, w, _ = coords.shape
        levels = len(pyramid)
        nch = levels * (2 * radius + 1) ** 2
        out = torch.empty((b, h, w, nch), dtype=torch.float32, device=coords.device)
        _lib.call('corr_lookup', coords.device, _lib.ptr_array(pyramid), _lib.ptr(coords), b, h, w, levels, radius,
                  _lib.ptr(out), nch)
        ctx.save_for_backward(coords, *pyramid)
        ctx.radius = radius
        return out

    @staticmethod
    def backward(ctx, grad_out):
        coords, *pyramid = ctx.saved_tensors
        b, h, w, _ = coords.shape
        levels = len(pyramid)
        grad_out = grad_out.contiguous()
        g_coords = torch.zeros_like(coords)
        g_pyr = [torch.zeros_like(p) for p in pyramid]
        _lib.call('corr_lookup_backward', coords.device, _lib.ptr_array(pyramid), _lib.ptr(coords), _lib.ptr(grad_out),
                  b, h, w, levels, ctx.radius, _lib.ptr(g_coords), _lib.ptr_array(g_pyr))
        return (g_coords, None) + tuple(g_pyr)


class _Upsample8(torch.autograd.Function):
    """SmallRAFT's training upsampling of an NHWC flow: forward = the graph's F.interpolate(scale_factor=8, 'bilinear')
    on its NCHW view, unchanged; backward = raft_b200_upflow8_backward, a gather in a fixed order.  PyTorch's own CUDA
    backward of that op scatters with atomics, and torch.use_deterministic_algorithms(True) refuses it."""

    @staticmethod
    def forward(ctx, flow):
        ctx.shape = flow.shape
        return F.interpolate(flow.permute(0, 3, 1, 2), scale_factor=8, mode='bilinear', align_corners=False)

    @staticmethod
    def backward(ctx, grad_up):
        b, h, w, _ = ctx.shape
        grad_up = grad_up.permute(0, 2, 3, 1).contiguous()
        grad_flow = torch.empty((b, h, w, 2), dtype=torch.float32, device=grad_up.device)
        _lib.call('upflow8_backward', grad_up.device, _lib.ptr(grad_up), b, h, w, _lib.ptr(grad_flow))
        return grad_flow


class _CorrPyramid(torch.autograd.Function):
    """CorrBlock.__init__: forward = the wgmma correlation kernels; backward = fp32 GEMMs on the pooled features
    (level l = fmap1 . avgpool^l(fmap2)^T / sqrt(C), so d fmap1 = sum_l dP_l . pool^l(fmap2) / sqrt(C) and
    d pool^l(fmap2) = dP_l^T . fmap1 / sqrt(C), un-pooled through the 2x2 means)."""

    @staticmethod
    def forward(ctx, fmap1, fmap2, levels, radius, precision):
        cb = CorrBlock(fmap1.detach(), fmap2.detach(), num_levels=levels, radius=radius, precision=precision)
        ctx.save_for_backward(fmap1, fmap2)
        ctx.levels = levels
        return tuple(cb.corr_pyramid)

    @staticmethod
    def backward(ctx, *g_pyr):
        fmap1, fmap2 = ctx.saved_tensors
        b, h, w, c = fmap1.shape
        scale = 1.0 / math.sqrt(c)
        f1 = fmap1.reshape(b, h * w, c)
        g1 = torch.zeros_like(f1)
        with torch.enable_grad():
            f2 = fmap2.detach().requires_grad_(True)
            pooled = [f2.permute(0, 3, 1, 2)]
            for _ in range(1, ctx.levels):
                pooled.append(F.avg_pool2d(pooled[-1], 2, 2))
            flat = [p.permute(0, 2, 3, 1).reshape(b, -1, c) for p in pooled]
        g_flat = []
        for l in range(ctx.levels):
            gp = g_pyr[l]
            if gp is None:
                g_flat.append(torch.zeros_like(flat[l]))
                continue
            gp = gp.reshape(b, h * w, -1)                                        # (b, q, n_l)
            g1 += torch.bmm(gp, flat[l].detach()) * scale
            g_flat.append(torch.bmm(gp.transpose(1, 2), f1) * scale)
        (g2,) = torch.autograd.grad(flat, f2, g_flat)
        return g1.reshape(fmap1.shape), g2, None, None, None


class _UnsupLoss(torch.autograd.Function):
    """UnsupervisedLoss on stacked predictions: forward = raft_b200_unsup_loss once per direction, which writes the loss
    terms and, in the same pass, the gradient of each direction's share of the loss with respect to every prediction;
    backward = that gradient scaled by grad_output.

    flows (2n, B, H, W, 2): the n forward predictions, then the n backward ones; census (2B, H, W, 48) and images
    (2B, H, W, 3): [image1; image2]; occ (2B, H, W) bool: [occ_fw; occ_bw]; census_norm: None (each direction divides
    its census sum by max(its mask count, 1)) or a device float64 (2,) tensor of the two directions' normalisers."""

    NPARTIALS = 4 * 1024              # fp64 scratch of a call: 4 per CTA (fixed, so that every call reduces alike)

    @staticmethod
    def forward(ctx, flows, census, images, occ, census_weight, smoothness_weight, edge_weight, gamma, census_norm=None):
        flows = flows.contiguous()
        n2, b, h, w, _ = flows.shape
        n = n2 // 2
        occ = occ.to(torch.uint8).contiguous()
        grad = torch.empty_like(flows)
        partials = torch.empty(_UnsupLoss.NPARTIALS, dtype=torch.float64, device=flows.device)
        sums = torch.empty((2, 4), dtype=torch.float64, device=flows.device)
        for d in range(2):                                     # d = 0: image1 -> image2, d = 1: image2 -> image1
            t, s = slice(d * b, (d + 1) * b), slice((1 - d) * b, (2 - d) * b)
            _lib.call('unsup_loss_norm', flows.device, _lib.ptr(census[t]), _lib.ptr(census[s]), _lib.ptr(images[t]),
                      _lib.ptr(occ[t]), _lib.ptr(flows[d * n:(d + 1) * n]), n, b, h, w, census_weight,
                      smoothness_weight, edge_weight, gamma, _lib.ptr(partials), partials.numel(), _lib.ptr(sums[d]),
                      _lib.ptr(grad[d * n:(d + 1) * n]), _lib.ptr(None if census_norm is None else census_norm[d]))
        ctx.save_for_backward(grad)
        ctx.terms = sums                                       # [direction][L_c, L_s, mask count, share of the loss]
        return (sums[0, 3] + sums[1, 3]).to(torch.float32)

    @staticmethod
    def backward(ctx, grad_out):
        (grad,) = ctx.saved_tensors
        return grad * grad_out, None, None, None, None, None, None, None, None


TRAIN_PRECISIONS = ('fp32', 'f16x2')


class _ConvTC(torch.autograd.Function):
    """A stride-1 Conv2D with odd, symmetric 'same' padding on the tensor cores (raft_b200_conv_tc_forward / _backward):
    x (B, cin, H, W) as a view of NHWC memory (torch.channels_last, read without a transpose), kernel HWIO, bias (cout,).
    The forward keeps the fp16 hi/lo planes of x for the backward, not x; the backward writes the kernel gradient and,
    when x needs one, the input gradient; the bias gradient is a torch reduction."""

    @staticmethod
    def forward(ctx, x, kernel, bias, workspaces):
        b, cin, h, w = x.shape
        kh, kw, _, cout = kernel.shape
        dims = (b, h, w, cin, kh, kw, cout)
        ws = workspaces.get(dims)
        if ws is None:
            need = ctypes.c_size_t()
            _lib.call('conv_tc_forward', x.device, None, None, None, *dims, None, None, None, ctypes.byref(need))
            ws = workspaces[dims] = _lib.workspace(need.value, x.device)
        x_nhwc = x.permute(0, 2, 3, 1).contiguous()
        kernel = kernel.detach().contiguous()
        planes = torch.empty(2 * b * h * w * ((cin + 63) // 64 * 64) + 128, dtype=torch.float16, device=x.device)
        out = torch.empty((b, h, w, cout), dtype=torch.float32, device=x.device)
        _lib.call('conv_tc_forward', x.device, _lib.ptr(x_nhwc), _lib.ptr(kernel), _lib.ptr(bias.detach().contiguous()),
                  *dims, _lib.ptr(out), _lib.ptr(planes), _lib.ptr(ws), ctypes.byref(ctypes.c_size_t(ws.numel())))
        ctx.save_for_backward(kernel)
        ctx.planes, ctx.ws, ctx.dims = planes, ws, dims
        return out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, grad_out):
        (kernel,) = ctx.saved_tensors
        b, h, w, cin, kh, kw, cout = ctx.dims
        g = grad_out.permute(0, 2, 3, 1).contiguous()
        grad_x = torch.empty((b, h, w, cin), dtype=torch.float32, device=g.device) if ctx.needs_input_grad[0] else None
        grad_kernel = torch.empty_like(kernel)
        _lib.call('conv_tc_backward', g.device, _lib.ptr(ctx.planes), _lib.ptr(kernel), _lib.ptr(g), *ctx.dims,
                  _lib.ptr(grad_x), _lib.ptr(grad_kernel), _lib.ptr(ctx.ws), ctypes.byref(ctypes.c_size_t(ctx.ws.numel())))
        grad_bias = g.sum(dim=(0, 1, 2)) if ctx.needs_input_grad[2] else None
        ctx.planes = None
        return None if grad_x is None else grad_x.permute(0, 3, 1, 2), grad_kernel, grad_bias, None


def _all_reduce_sum(x):
    """differentiable all-reduce (sum) over the default process group; identity without one."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        import torch.distributed.nn.functional as dnf
        return dnf.all_reduce(x, op=dist.ReduceOp.SUM)
    return x


class TrainGraph:
    """The forward of model.py:68-109 / 190-226 with `training=True` in backward-capable form, on leaf parameters `P`
    (HWIO kernels, reference attribute paths).  NCHW inside, NHWC at the interface."""

    def __init__(self, P, variant, precision, moving, train_precision='fp32'):
        self.P, self.variant, self.precision, self.moving = P, variant, precision, moving
        self.train_precision = train_precision
        self._conv_ws = {}                              # _ConvTC workspaces by shape
        self.cfg = dict(raft=dict(hidden=128, context=128, levels=4, radius=4, fnorm='instance', cnorm='batch'),
                        small=dict(hidden=96, context=64, levels=4, radius=3, fnorm='instance', cnorm=None))[variant]

    # -- primitives --
    def conv(self, x, name, stride=1, padding='same'):
        if self.train_precision == 'f16x2':
            return self._conv_f16x2(x, name, stride, padding)
        return self._conv_lib(x, name, stride, padding)

    def _conv_lib(self, x, name, stride, padding):
        w = self.P[name + '.kernel'].permute(3, 2, 0, 1)
        if padding == 'same':
            pt, pb = _same_pads(x.shape[2], w.shape[2], stride)
            pl, pr = _same_pads(x.shape[3], w.shape[3], stride)
            if pt or pb or pl or pr:
                x = F.pad(x, (pl, pr, pt, pb))
        return F.conv2d(x, w, self.P[name + '.bias'], stride=stride)

    def _conv_f16x2(self, x, name, stride, padding):
        """train_precision='f16x2': stride 1, 'same' (odd kernel) or 1x1 'valid', cin >= 64 on the tensor cores; convf1
        (cin 2), SmallRAFT's 32-channel first stage, the stems and the stride-2 convolutions on the library, their outputs
        put back into channels_last.  A 32-channel layer would fill half of the one 64-channel chunk it is padded to, and
        its weight gradients, behind an instance norm at the full resolution of SmallRAFT's first stage, leave the
        IEEE-fp32 gradient gates of the step on the three-pass split (DESIGN.md section 9.0)."""
        kernel = self.P[name + '.kernel']
        kh, kw, cin, _ = kernel.shape
        if stride == 1 and cin >= 64 and kh % 2 == 1 and kw % 2 == 1 and (padding == 'same' or kh == kw == 1):
            return _ConvTC.apply(x, kernel, self.P[name + '.bias'], self._conv_ws)
        return self._conv_lib(x, name, stride, padding).contiguous(memory_format=torch.channels_last)

    def norm(self, x, name, norm_type):
        eps = 1e-3
        if norm_type is None:
            return x
        g = self.P[name + '.gamma'].view(1, -1, 1, 1)
        b = self.P[name + '.beta'].view(1, -1, 1, 1)
        if norm_type == 'instance':
            mean = x.mean(dim=(2, 3), keepdim=True)
            var = x.var(dim=(2, 3), unbiased=False, keepdim=True)
        else:                                           # batch statistics over the GLOBAL batch (all ranks)
            n_local = x.shape[0] * x.shape[2] * x.shape[3]
            stats = torch.stack([x.sum(dim=(0, 2, 3)), (x * x).sum(dim=(0, 2, 3))])
            stats = _all_reduce_sum(stats)
            n = n_local * (dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1)
            mean = (stats[0] / n).view(1, -1, 1, 1)
            var = (stats[1] / n).view(1, -1, 1, 1) - mean * mean
            with torch.no_grad():                       # keras moving statistics, momentum 0.99 (DESIGN.md §9)
                mom = 0.99
                self.moving[name + '.moving_mean'].mul_(mom).add_((1 - mom) * mean.flatten())
                self.moving[name + '.moving_variance'].mul_(mom).add_((1 - mom) * n / max(n - 1, 1) * var.flatten())
        return (x - mean) * torch.rsqrt(var + eps) * g + b

    def res_block(self, x, p, nt, stride):
        fx = F.relu(self.norm(self.conv(x, p + '.conv1', stride), p + '.norm1', nt))
        fx = F.relu(self.norm(self.conv(fx, p + '.conv2', 1), p + '.norm2', nt))
        if stride != 1:
            x = self.norm(self.conv(x, p + '.downsample.0', stride, padding='valid'), p + '.downsample.1', nt)
        return F.relu(x + fx)

    def encoder(self, x, prefix, nt):
        x = F.relu(self.norm(self.conv(x, prefix + '.conv1', 2), prefix + '.norm1', nt))
        for li, s in ((1, 1), (2, 2), (3, 2)):
            x = self.res_block(x, f'{prefix}.layer{li}.0', nt, s)
            x = self.res_block(x, f'{prefix}.layer{li}.1', nt, 1)
        return self.conv(x, prefix + '.conv2', 1, padding='valid')

    def gru_pass(self, h, x, prefix, s):
        hx = torch.cat([h, x], dim=1)
        z = torch.sigmoid(self.conv(hx, prefix + '.convz' + s))
        r = torch.sigmoid(self.conv(hx, prefix + '.convr' + s))
        q = torch.tanh(self.conv(torch.cat([r * h, x], dim=1), prefix + '.convq' + s))
        return (1 - z) * h + z * q

    def update_block(self, net, inp, corr, flow):
        e, u = 'update_block.encoder', 'update_block'
        if self.variant == 'raft':
            cor = F.relu(self.conv(corr, e + '.convc1', padding='valid'))
            cor = F.relu(self.conv(cor, e + '.convc2'))
        else:
            cor = F.relu(self.conv(corr, e + '.convc1'))
        flo = F.relu(self.conv(flow, e + '.convf1'))
        flo = F.relu(self.conv(flo, e + '.convf2'))
        out = F.relu(self.conv(torch.cat([cor, flo], dim=1), e + '.conv'))
        x = torch.cat([inp, out, flow], dim=1)
        if self.variant == 'raft':
            net = self.gru_pass(net, x, u + '.gru', '1')
            net = self.gru_pass(net, x, u + '.gru', '2')
        else:
            net = self.gru_pass(net, x, u + '.gru', '')
        delta = self.conv(F.relu(self.conv(net, u + '.flow_head.conv1')), u + '.flow_head.conv2')
        mask = None
        if self.variant == 'raft':
            mask = 0.25 * self.conv(F.relu(self.conv(net, u + '.mask.0')), u + '.mask.2', padding='valid')
        return net, mask, delta

    @staticmethod
    def upsample_flow(flow, mask):
        """model.py:39-66 on NHWC."""
        bs, h, w, _ = flow.shape
        m = torch.softmax(mask.reshape(bs, h, w, 8, 8, 9, 1), dim=5)
        f = F.pad(8 * flow, (0, 0, 1, 1, 1, 1))
        patches = torch.stack([f[:, ky:ky + h, kx:kx + w, :] for ky in range(3) for kx in range(3)], dim=3)
        up = (m * patches.reshape(bs, h, w, 1, 1, 9, 2)).sum(dim=5)
        return up.permute(0, 1, 3, 2, 4, 5).reshape(bs, 8 * h, 8 * w, 2)

    def forward(self, image1, image2, iters):
        cfg = self.cfg
        bs, H, W, _ = image1.shape
        x1 = 2 * (image1 / 255.0) - 1.0
        x2 = 2 * (image2 / 255.0) - 1.0
        both = torch.cat([x1, x2], dim=0).permute(0, 3, 1, 2)
        fm = self.encoder(both, 'fnet', cfg['fnorm']).permute(0, 2, 3, 1)
        fmap1, fmap2 = fm[:bs].contiguous(), fm[bs:].contiguous()
        pyramid = _CorrPyramid.apply(fmap1, fmap2, cfg['levels'], cfg['radius'], self.precision)
        cnet = self.encoder(x1.permute(0, 3, 1, 2), 'cnet', cfg['cnorm'])
        return self._iterate(pyramid, cnet, bs, H, W, iters, image1.device)

    def forward_bidirectional(self, image1, image2, iters):
        """Both directions of B pairs as one graph: fnet and cnet each run once on [x1; x2], and the loop runs at batch
        2B with fmap1 = [f1; f2], fmap2 = [f2; f1], as `RAFT.predict_bidirectional` does.  Returns (preds_fw, preds_bw),
        the n predictions image1 -> image2 and image2 -> image1, each (B, H, W, 2).

        One consequence: cnet's BatchNorm (RAFT) normalises over, and updates its moving statistics from, the 2B images
        -- the global 2B under torch.distributed (SyncBN) -- where the supervised step's sees image1 only."""
        cfg = self.cfg
        bs, H, W, _ = image1.shape
        x1 = 2 * (image1 / 255.0) - 1.0
        x2 = 2 * (image2 / 255.0) - 1.0
        both = torch.cat([x1, x2], dim=0).permute(0, 3, 1, 2)
        fm = self.encoder(both, 'fnet', cfg['fnorm']).permute(0, 2, 3, 1)
        fmap1, fmap2 = fm.contiguous(), torch.cat([fm[bs:], fm[:bs]]).contiguous()
        pyramid = _CorrPyramid.apply(fmap1, fmap2, cfg['levels'], cfg['radius'], self.precision)
        cnet = self.encoder(both, 'cnet', cfg['cnorm'])
        preds = self._iterate(pyramid, cnet, 2 * bs, H, W, iters, image1.device)
        return [p[:bs] for p in preds], [p[bs:] for p in preds]

    def _iterate(self, pyramid, cnet, bs, H, W, iters, device):
        """model.py:86-106: the context split and `iters` update-block iterations from zero flow; the upsampled
        predictions."""
        cfg = self.cfg
        net = torch.tanh(cnet[:, :cfg['hidden']])
        inp = F.relu(cnet[:, cfg['hidden']:])
        h, w = H // 8, W // 8
        gy, gx = torch.meshgrid(torch.arange(h, dtype=torch.float32, device=device),
                                torch.arange(w, dtype=torch.float32, device=device), indexing='ij')
        coords0 = torch.stack([gx, gy], dim=-1)[None].repeat(bs, 1, 1, 1)
        coords1 = coords0.clone()
        preds = []
        for _ in range(iters):
            corr = _Lookup.apply(coords1, cfg['radius'], *pyramid)
            flow = coords1 - coords0
            net, mask, delta = self.update_block(net, inp, corr.permute(0, 3, 1, 2), flow.permute(0, 3, 1, 2))
            coords1 = coords1 + delta.permute(0, 2, 3, 1)
            if self.variant == 'raft':
                preds.append(self.upsample_flow(coords1 - coords0, mask.permute(0, 2, 3, 1)))
            elif coords1.is_cuda:
                preds.append(8 * _Upsample8.apply(coords1 - coords0).permute(0, 2, 3, 1))
            else:
                up = F.interpolate((coords1 - coords0).permute(0, 3, 1, 2), scale_factor=8, mode='bilinear', align_corners=False)
                preds.append(8 * up.permute(0, 2, 3, 1))
        return preds


class Trainer:
    """State of `RAFT.train_step`: flat parameters / moments, the backward-capable graph, the step itself."""

    def __init__(self, model):
        self.model = model
        self.variant = 'raft' if model._variant == _lib.VARIANT_BASIC else 'small'
        sd = model.state_dict()
        self.flat = FlatState(sd, lambda k: not (k.endswith('.moving_mean') or k.endswith('.moving_variance')))
        self.moving = {k: v.clone() for k, v in sd.items() if k.endswith('.moving_mean') or k.endswith('.moving_variance')}
        self.graph = TrainGraph(self.flat.views, self.variant, model.precision, self.moving, model.train_precision)
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1

    def params(self):
        out = {k: v.detach() for k, v in self.flat.views.items()}
        out.update(self.moving)
        return out

    def step(self, data, optimizer, clip_norm, loss_fn=sequence_loss, epe_fn=end_point_error):
        if isinstance(loss_fn, UnsupervisedLoss):
            return self._step_unsupervised(data, optimizer, clip_norm, loss_fn, epe_fn)
        image1, image2, flow_gt, valid = data
        image1 = image1.to(torch.float32)
        image2 = image2.to(torch.float32)
        self.flat.zero_grad()
        # cuDNN off for the forward AND the backward of the step: on the H100 its algorithm choice for the small encoder's
        # convolutions gives feature-encoder gradients ~10x further from an IEEE-fp32 autograd step than PyTorch's own
        # (im2col + IEEE GEMM) convolutions -- up to 5 % of a tensor's largest entry (tests/test_train.py).
        cudnn_enabled = torch.backends.cudnn.enabled
        torch.backends.cudnn.enabled = False
        try:
            preds = self.graph.forward(image1, image2, self.model.iters)       # model.py:131 (training=True)
            loss = loss_fn([flow_gt, valid], preds)                            # :132
            # tape.gradient (:133).  Each rank's loss is the mean over ITS shard: the mean over the global batch is the
            # average of the shard means (equal shard sizes), so gradients are summed over ranks and divided by the world
            # size.
            loss.backward()
        finally:
            torch.backends.cudnn.enabled = cudnn_enabled
        if self.world > 1:
            dist.all_reduce(self.flat.g, op=dist.ReduceOp.SUM)                 # ONE flat NCCL all-reduce per step
            self.flat.g.div_(self.world)
        self.flat.apply(optimizer, clip_norm)                                  # :135-136
        with torch.no_grad():
            info = epe_fn([flow_gt, valid], preds[-1].detach())                # :138
        return loss.detach(), info

    def _step_unsupervised(self, data, optimizer, clip_norm, loss_fn, epe_fn):
        """`step` with an UnsupervisedLoss: the bidirectional graph, the loss on both directions' predictions, then the
        same all-reduce, clipping and AdamW.  data = (image1, image2) or (image1, image2, flow, valid); with ground truth
        the metrics are taken on the forward final prediction, without it they are None."""
        if len(data) not in (2, 4):
            raise ValueError(f'unsupervised train_step takes (image1, image2[, flow, valid]); got {len(data)} items')
        image1 = data[0].to(torch.float32)
        image2 = data[1].to(torch.float32)
        self.flat.zero_grad()
        cudnn_enabled = torch.backends.cudnn.enabled                     # off, as in the supervised step
        torch.backends.cudnn.enabled = False
        try:
            preds = self.graph.forward_bidirectional(image1, image2, self.model.iters)
            loss = loss_fn((image1, image2), preds)
            loss.backward()
        finally:
            torch.backends.cudnn.enabled = cudnn_enabled
        if self.world > 1:
            dist.all_reduce(self.flat.g, op=dist.ReduceOp.SUM)
            self.flat.g.div_(self.world)
        self.flat.apply(optimizer, clip_norm)
        info = None
        if len(data) == 4:
            with torch.no_grad():
                info = epe_fn([data[2], data[3]], preds[0][-1].detach())
        return loss.detach(), info
