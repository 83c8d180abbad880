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
  through torch.autograd, with cuDNN switched off for the step (see Trainer.step) -- library code, stated as such; the
  hand-written tensor-core kernels are forward-only.
"""
import math
import os

import numpy as np
import torch
import torch.distributed as dist
import torch.nn.functional as F

from . import _lib
from .datasets.flow_viz import flow_to_image
from .datasets.frame_utils import write_png
from .layers.corr import CorrBlock
from .layers.extractor import _same_pads, force_ieee_fp32
from .losses import end_point_error, sequence_loss
from .preprocess import resize_with_crop_or_pad

force_ieee_fp32()


# ------------------------------------------------------------------------------------------------ schedules / optimiser
def first_cycle_scaler(cycle):
    """tf_raft/training.py:10-15: 1 during the first cycle, 0 afterwards (min_lr -> max_lr -> min_lr -> const)."""
    return 1.0 if cycle == 1 else 0.0


def inverse_scaler(cycle):
    """tf_raft/training.py:18-23."""
    return 1.0 / cycle


class VisFlowCallback:
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

    def set_model(self, model):
        self.model = model

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

    def zero_grad(self):
        self.g.zero_()

    def global_norm(self):
        """sqrt(sum g^2) over every trainable variable (tf.linalg.global_norm), on the device."""
        with torch.cuda.device(self.g.device):
            _lib.check(_lib.lib().raft_b200_sumsq(_lib.ptr(self.g), self.g.numel(), _lib.ptr(self._part), self._part.numel(),
                                                  _lib.ptr(self._norm), _lib.stream()), 'sumsq')
        return self._norm                                                    # device scalar: sum of squares

    def apply(self, opt, clip_norm):
        """clip_by_global_norm (model.py:135) + AdamW apply_gradients (:136), one launch; no host synchronisation."""
        sumsq = self.global_norm()
        opt.iterations += 1
        t = opt.iterations
        lr = opt.lr() if not callable(opt.learning_rate) else float(opt.learning_rate(t - 1))
        lr_t = lr * math.sqrt(1 - opt.beta_2 ** t) / (1 - opt.beta_1 ** t)
        with torch.cuda.device(self.g.device):
            _lib.check(_lib.lib().raft_b200_adamw_step(
                _lib.ptr(self.p), _lib.ptr(self.g), _lib.ptr(self.m), _lib.ptr(self.v), self.p.numel(), _lib.ptr(sumsq),
                float(clip_norm if clip_norm else 0.0), float(lr_t), float(opt.beta_1), float(opt.beta_2),
                float(opt.epsilon), float(opt.weight_decay), _lib.stream()), 'adamw_step')


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
        with torch.cuda.device(coords.device):
            _lib.check(_lib.lib().raft_b200_corr_lookup(_lib.ptr_array(pyramid), _lib.ptr(coords), b, h, w, levels, radius,
                                                        _lib.ptr(out), nch, _lib.stream()), 'corr_lookup')
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
        with torch.cuda.device(coords.device):
            _lib.check(_lib.lib().raft_b200_corr_lookup_backward(
                _lib.ptr_array(pyramid), _lib.ptr(coords), _lib.ptr(grad_out), b, h, w, levels, ctx.radius,
                _lib.ptr(g_coords), _lib.ptr_array(g_pyr), _lib.stream()), 'corr_lookup_backward')
        return (g_coords, None) + tuple(g_pyr)


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


def _all_reduce_sum(x):
    """differentiable all-reduce (sum) over the default process group; identity without one."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        import torch.distributed.nn.functional as dnf
        return dnf.all_reduce(x, op=dist.ReduceOp.SUM)
    return x


class TrainGraph:
    """The forward of model.py:68-109 / 190-226 with `training=True` in backward-capable form, on leaf parameters `P`
    (HWIO kernels, reference attribute paths).  NCHW inside, NHWC at the interface."""

    def __init__(self, P, variant, precision, moving):
        self.P, self.variant, self.precision, self.moving = P, variant, precision, moving
        self.cfg = dict(raft=dict(hidden=128, context=128, levels=4, radius=4, fnorm='instance', cnorm='batch'),
                        small=dict(hidden=96, context=64, levels=4, radius=3, fnorm='instance', cnorm=None))[variant]

    # -- primitives --
    def conv(self, x, name, stride=1, padding='same'):
        w = self.P[name + '.kernel'].permute(3, 2, 0, 1)
        if padding == 'same':
            pt, pb = _same_pads(x.shape[2], w.shape[2], stride)
            pl, pr = _same_pads(x.shape[3], w.shape[3], stride)
            if pt or pb or pl or pr:
                x = F.pad(x, (pl, pr, pt, pb))
        return F.conv2d(x, w, self.P[name + '.bias'], stride=stride)

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
        net = torch.tanh(cnet[:, :cfg['hidden']])
        inp = F.relu(cnet[:, cfg['hidden']:])
        h, w = H // 8, W // 8
        gy, gx = torch.meshgrid(torch.arange(h, dtype=torch.float32, device=image1.device),
                                torch.arange(w, dtype=torch.float32, device=image1.device), indexing='ij')
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
        self.graph = TrainGraph(self.flat.views, self.variant, model.precision, self.moving)
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1

    def params(self):
        out = {k: v.detach() for k, v in self.flat.views.items()}
        out.update(self.moving)
        return out

    def step(self, data, optimizer, clip_norm, loss_fn=sequence_loss, epe_fn=end_point_error):
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
