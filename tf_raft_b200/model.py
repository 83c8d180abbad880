"""RAFT / SmallRAFT -- host-side mirror of tf_raft/model.py.

`RAFT(drop_rate=0, iters=12, iters_pred=24)([image1, image2], training)` returns the list of
`iters` (training) or `iters_pred` (inference) flow predictions (B, H, W, 2), like the reference
(model.py:68-109 / 190-226).  The whole iteration loop (lookup -> update block -> coords += delta ->
upsample) is ONE call into libraft_b200.so (raft_b200_forward_loop); the correlation pyramid is
another (raft_b200_corr_pyramid_build); in inference on the native encoders, so are the encoders, run as concurrent
stream branches (raft_b200_encode_pair).  Optionally the whole forward is replayed from a CUDA graph.
"""
from collections import OrderedDict

import numpy as np
import torch

from . import _lib
from .layers.corr import CorrBlock, coords_grid, coords_init, fb_occlusion, forward_interpolate, upflow8
from .layers.extractor import BasicEncoder, SmallEncoder
from .layers.update import BasicUpdateBlock, SmallUpdateBlock
from .losses import end_point_error, sequence_loss


class RAFT:
    _variant = _lib.VARIANT_BASIC

    def __init__(self, drop_rate=0, iters=12, iters_pred=24, *, precision=None, device='cuda', seed=None,
                 use_graph=False, encoder_backend=None, **kwargs):
        self.hidden_dim = 128
        self.context_dim = 128
        self.corr_levels = 4
        self.corr_radius = 4
        self.drop_rate = drop_rate
        self.iters = iters
        self.iters_pred = iters_pred
        self.precision = _lib.resolve_precision(precision)
        self.device = torch.device(device)
        self.use_graph = use_graph
        self.encoder_backend = encoder_backend
        self._build_layers(seed)
        self._graphs = {}
        self._pair_ws = _lib.WorkspaceCache()
        self.flow_metrics = None
        self.optimizer = None
        self.train_precision = 'fp32'
        self._trainer = None
        self._params_stale = False
        self._pending_slots = None                         # optimiser state of load_weights awaiting the Trainer

    def _encoder_backend(self):
        # the all-FFMA reference configuration keeps cuDNN IEEE-fp32 encoders; the product path is native
        return self.encoder_backend or ('native' if self.precision == _lib.PREC_F16X2 else 'torch')

    def _build_layers(self, seed):
        s = 0 if seed is None else seed
        self.fnet = BasicEncoder(output_dim=256, norm_type='instance', drop_rate=self.drop_rate, device=self.device,
                                 seed=s, backend=self._encoder_backend())
        self.cnet = BasicEncoder(output_dim=self.hidden_dim + self.context_dim, norm_type='batch',
                                 drop_rate=self.drop_rate, device=self.device, seed=s + 1, backend=self._encoder_backend())
        self.update_block = BasicUpdateBlock(filters=self.hidden_dim, precision=self.precision, device=self.device,
                                             seed=s + 2)

    # -- parameters ---------------------------------------------------------------------------
    def load_params(self, params):
        """`{'fnet.conv1.kernel': ..., 'cnet....', 'update_block.encoder.convc1.kernel': ...}` (NumPy or torch)."""
        self.fnet.load_params(params, 'fnet.')
        self.cnet.load_params(params, 'cnet.')
        self.update_block.load_params(params, 'update_block.')
        self._graphs.clear()
        self._trainer = None                               # a training state built on the old values is void
        self._params_stale = False
        self._pending_slots = None

    def save_weights(self, filepath):
        """Keras's `model.save_weights(filepath)` in its TensorFlow format: a tensor bundle at prefix `filepath`
        (`filepath.index`, `filepath.data-00000-of-00001`) whose keys are the reference's object-graph keys
        (`checkpoint.param_to_tf_key`), BatchNorm moving statistics included.  Once `train_step` has run (or optimiser
        state was loaded), Adam's moments are saved under `<variable>/.OPTIMIZER_SLOT/optimizer/m|v/...` and the step
        count under `optimizer/iter` (int64), so that `load_weights` resumes the run.

        Not written: TensorFlow's `_CHECKPOINTABLE_OBJECT_GRAPH` proto.  `load_weights` and `load_tf_checkpoint` here
        read these files; TensorFlow's own `load_weights` needs that proto and cannot."""
        from .checkpoint import OPTIMIZER_ITER_KEY, optimizer_slot_key, param_to_tf_key, write_tf_checkpoint
        tensors = {param_to_tf_key(k): v.detach().cpu().numpy() for k, v in self.state_dict().items()}
        slots = self._pending_slots
        if self._trainer is not None:
            flat = self._trainer.flat
            slots = {'iter': self.optimizer.iterations}
            for name, buf in (('m', flat.m), ('v', flat.v)):
                host = buf.cpu()
                slots[name] = {k: view.numpy() for k, view in flat.slot(host).items()}
        if slots is not None:
            for name in ('m', 'v'):
                tensors.update((optimizer_slot_key(k, name), a) for k, a in slots[name].items())
            tensors[OPTIMIZER_ITER_KEY] = np.array(slots['iter'], dtype=np.int64)
        write_tf_checkpoint(filepath, tensors)

    def load_weights(self, filepath):
        """Loads what `save_weights` (or a TensorFlow-written tensor bundle with the reference's keys) holds at prefix
        `filepath`: the parameters through `load_tf_checkpoint(filepath, expect=self.state_dict())`.  When the file also
        holds Adam's moments of every trainable variable and `optimizer/iter`, they are applied when the training state
        is built -- at once if `compile` has run, else at `compile` -- and `optimizer.iterations` is set, so the
        learning-rate schedule continues where the saved run stopped (the reference's `resume`).  Without them only
        the weights load."""
        from .checkpoint import OPTIMIZER_ITER_KEY, load_tf_checkpoint, optimizer_slot_key, read_tf_checkpoint
        self.load_params(load_tf_checkpoint(filepath, expect=self.state_dict()))
        tensors = read_tf_checkpoint(filepath)
        shapes = {k: tuple(v.shape) for k, v in self.state_dict().items()
                  if not (k.endswith('.moving_mean') or k.endswith('.moving_variance'))}
        keys = {(k, name): optimizer_slot_key(k, name) for k in shapes for name in ('m', 'v')}
        found = [key for key in keys.values() if key in tensors]
        if not found and OPTIMIZER_ITER_KEY not in tensors:
            return
        missing = [key for key in keys.values() if key not in tensors]
        if OPTIMIZER_ITER_KEY not in tensors:
            missing.append(OPTIMIZER_ITER_KEY)
        bad = [key for (k, _), key in keys.items() if key in tensors and tuple(tensors[key].shape) != shapes[k]]
        if missing or bad:
            raise ValueError(f'{filepath}: incomplete optimiser state -- missing {missing[:4]}'
                             f'{"..." if len(missing) > 4 else ""}, mis-shaped {bad[:4]}')
        self._pending_slots = {'iter': int(tensors[OPTIMIZER_ITER_KEY]),
                               'm': {k: tensors[keys[k, 'm']] for k in shapes},
                               'v': {k: tensors[keys[k, 'v']] for k in shapes}}
        if self.optimizer is not None:
            self._build_trainer()

    def _build_trainer(self):
        """The training state of `train_step`, with the optimiser state `load_weights` left pending applied to it."""
        from .train import AdamW, Trainer
        if not isinstance(self.optimizer, AdamW):
            raise TypeError('optimizer must be tf_raft_b200.train.AdamW (tfa.optimizers.AdamW semantics)')
        self._trainer = Trainer(self)
        slots, self._pending_slots = self._pending_slots, None
        if slots is not None:
            flat = self._trainer.flat
            for name, buf in (('m', flat.m), ('v', flat.v)):
                for k, view in flat.slot(buf).items():
                    view.copy_(torch.from_numpy(np.ascontiguousarray(slots[name][k], dtype=np.float32)))
            self.optimizer.iterations = slots['iter']

    def state_dict(self):
        self._sync_trained_params()
        out = OrderedDict()
        out.update(self.fnet.state_dict('fnet.'))
        out.update(self.cnet.state_dict('cnet.'))
        out.update(self.update_block.state_dict('update_block.'))
        return out

    # -- reference helpers ----------------------------------------------------------------------
    def initialize_flow(self, image):
        """model.py:32-37: coords0 = coords1 = coords_grid(B, H//8, W//8)."""
        bs, h, w, _ = image.shape
        return coords_grid(bs, h // 8, w // 8, self.device), coords_grid(bs, h // 8, w // 8, self.device)

    def upsample_flow(self, flow, mask):
        """model.py:39-66: convex 8x upsampling."""
        flow, mask = _lib.f32c(flow), _lib.f32c(mask)
        b, h, w, _ = flow.shape
        if tuple(mask.shape) != (b, h, w, 576):
            raise ValueError(f'mask: expected {(b, h, w, 576)}, got {tuple(mask.shape)}')
        out = torch.empty((b, 8 * h, 8 * w, 2), dtype=torch.float32, device=flow.device)
        _lib.call('upsample_convex', flow.device, _lib.ptr(flow), _lib.ptr(mask), b, h, w, _lib.ptr(out))
        return out

    # -- forward ----------------------------------------------------------------------------------
    def _encode(self, image1, image2, training):
        # model.py:70-71 (2*(x/255)-1) happens inside the encoders' first load (raw_image=True)
        if not training and self.fnet.backend == self.cnet.backend == 'native':
            return self._encode_pair(image1, image2)
        fmap1, fmap2 = self.fnet([image1, image2], training=training, raw_image=True)     # :74
        net, inp = self._context(image1, training)
        return fmap1, fmap2, net, inp

    def _context(self, image1, training):
        cnet = self.cnet(image1, training=training, raw_image=True)                       # :82
        b, h, w, _ = cnet.shape
        net = torch.empty((b, h, w, self.hidden_dim), dtype=torch.float32, device=cnet.device)
        inp = torch.empty((b, h, w, self.context_dim), dtype=torch.float32, device=cnet.device)
        _lib.call('context_split', cnet.device, _lib.ptr(cnet), b * h * w, self.hidden_dim, self.context_dim,
                  _lib.ptr(net), _lib.ptr(inp))                                           # :84-86
        return net, inp

    def _encode_pair(self, image1, image2):
        """The inference encode on the native encoders as one call, raft_b200_encode_pair: fnet(image1), fnet(image2)
        and cnet(image1) run as concurrent branches (one branch's norm and im2col passes overlap another's
        convolutions).  Every image's encoder output is independent of the batch it runs in, so this computes the bytes
        of the separate fnet([image1, image2]) and `_context(image1)` calls.  Returns (fmap1, fmap2, net, inp)."""
        bs, H, W, _ = image1.shape
        h, w = -(-H // 8), -(-W // 8)
        dev = image1.device
        ws = self._pair_ws.get((bs, H, W), dev, lambda: _lib.query_bytes(
            'encode_pair_workspace_bytes', self._variant, bs, H, W, self.hidden_dim + self.context_dim))
        fmap1 = torch.empty((bs, h, w, self.fnet.output_dim), dtype=torch.float32, device=dev)
        fmap2 = torch.empty_like(fmap1)
        net = torch.empty((bs, h, w, self.hidden_dim), dtype=torch.float32, device=dev)
        inp = torch.empty((bs, h, w, self.context_dim), dtype=torch.float32, device=dev)
        fnet, cnet = self.fnet, self.cnet
        # The call joins its side streams back into the current stream before it returns, so the tensors above (allocated
        # on the current stream) need no record_stream.
        _lib.call('encode_pair', dev, self._variant, _lib.ptr(fnet.prepared()), _lib.NORM_TYPES[fnet.norm_type],
                  fnet.output_dim, _lib.ptr(cnet.prepared()), _lib.NORM_TYPES[cnet.norm_type], self.hidden_dim,
                  self.context_dim, _lib.ptr(image1), _lib.ptr(image2), bs, H, W, _lib.ptr(fmap1), _lib.ptr(fmap2),
                  _lib.ptr(net), _lib.ptr(inp), _lib.ptr(ws), ws.numel())
        return fmap1, fmap2, net, inp

    def _loop(self, corr_block, net, inp, coords1, flow_ups, b, h, w):
        ub = self.update_block
        ws = ub.workspace(b, h, w)
        _lib.call('forward_loop', net.device, self._variant, _lib.ptr(ub.prepared()),
                  _lib.ptr_array(corr_block.corr_pyramid), self.corr_levels, self.corr_radius, _lib.ptr(net), _lib.ptr(inp),
                  _lib.ptr(coords1), _lib.ptr_array(flow_ups), len(flow_ups), b, h, w, _lib.ptr(ws), ws.numel(),
                  self.precision)

    def __call__(self, inputs, training, *, last_only=False, flow_init=None):
        """inputs = [image1, image2], each (B, H, W, 3) float in 0..255 on the GPU.

        `training` is required, as in the reference (model.py:68).  `last_only=True` (keyword-only
        extra) computes just the final prediction -- what predict_step returns (model.py:166).
        `flow_init` (keyword-only extra; tf-raft has no warm start): a (B, H/8, W/8, 2) float32 tensor on the images'
        device.  The loop then starts from coords1 = coords0 + flow_init (raft_b200_coords_init) instead of zero flow:
        RAFT's warm start, usually `forward_interpolate` of the previous pair's low-resolution flow (predict_video).
        With `use_graph=True` the whole forward of a given input shape is captured once into a CUDA graph
        and replayed; the returned tensors are then static buffers that the next call overwrites.  `flow_init` is then
        one more static input, copied in before each replay; warm and cold calls never share a graph."""
        image1, image2 = inputs
        image1, image2 = _lib.f32c(image1), _lib.f32c(image2)
        if flow_init is not None:
            flow_init = self._check_flow_init(flow_init, image1)
        self._sync_trained_params()
        if self.use_graph and not training:
            key = (tuple(image1.shape), bool(last_only), flow_init is not None)
            return self._graph_run(key, lambda a, b, f: self._forward(a, b, False, last_only, f),
                                   (image1, image2, flow_init))
        return self._forward(image1, image2, training, last_only, flow_init)

    @staticmethod
    def _check_flow_init(flow_init, image):
        if not isinstance(flow_init, torch.Tensor):
            raise TypeError(f'flow_init must be a torch tensor, got {type(flow_init).__name__}')
        if flow_init.dtype != torch.float32:
            raise TypeError(f'flow_init must be float32, got {flow_init.dtype}')
        if flow_init.device != image.device:
            raise ValueError(f'flow_init is on {flow_init.device}, the images on {image.device}')
        bs, H, W, _ = image.shape
        want = (bs, H // 8, W // 8, 2)
        if tuple(flow_init.shape) != want:
            raise ValueError(f'flow_init: expected {want} for {H}x{W} images, got {tuple(flow_init.shape)}')
        return flow_init.contiguous()

    def _graph_run(self, key, fn, inputs):
        """fn(*inputs) captured once per `key` into a CUDA graph over static copies of `inputs` (None entries stay
        None), then replayed: each call copies its inputs into the static ones and returns the captured outputs."""
        entry = self._graphs.get(key)
        if entry is None:
            statics = [None if t is None else t.clone() for t in inputs]
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(side):                      # warm-up: allocations, attributes, weight packing
                for _ in range(2):
                    fn(*statics)
            torch.cuda.current_stream(self.device).wait_stream(side)
            torch.cuda.synchronize(self.device)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                outs = fn(*statics)
            # The captured kernels hold raw addresses of the encoder / update-block workspaces; those caches keep one
            # shape at a time, so the graph entry owns references to the buffers it was captured with.
            keep = [c.buffers() for c in (self.fnet.workspaces, self.cnet.workspaces, self.update_block.workspaces,
                                            self._pair_ws)]
            entry = (graph, statics, outs, self._last, keep)
            self._graphs[key] = entry
        graph, statics, outs, last, _keep = entry
        for s, t in zip(statics, inputs):
            if t is not None:
                s.copy_(t, non_blocking=True)
        graph.replay()
        self._last = last
        return outs

    @staticmethod
    def _check_size(H, W):
        if H % 8 or W % 8:
            raise ValueError(f'image height and width must be multiples of 8 (got {H}x{W}); the reference fails in '
                             'update.py:146 for other sizes -- crop-or-pad first (datasets/dataset.py:323-334)')

    def _forward(self, image1, image2, training, last_only, flow_init=None):
        bs, H, W, _ = image1.shape
        self._check_size(H, W)
        fmap1, fmap2, net, inp = self._encode(image1, image2, training)
        return self._iterate(fmap1, fmap2, net, inp, bs, H, W, training, last_only, flow_init)

    def _iterate(self, fmap1, fmap2, net, inp, bs, H, W, training, last_only, flow_init):
        """Everything after the encoders: pyramid, entry state, iteration loop (model.py:77-106)."""
        h, w = H // 8, W // 8
        iters = self.iters if training else self.iters_pred                  # model.py:92
        corr_block = CorrBlock(fmap1, fmap2, num_levels=self.corr_levels, radius=self.corr_radius,
                               precision=self.precision)                      # :77-79
        if flow_init is None:
            coords1 = coords_grid(bs, h, w, self.device)                      # :89
        else:
            coords1 = coords_init(flow_init)                                  # :89 plus the warm start's initial flow
        preds = [torch.empty((bs, H, W, 2), dtype=torch.float32, device=self.device)
                 if (not last_only or i == iters - 1) else None for i in range(iters)]
        if iters:
            self._loop(corr_block, net, inp, coords1, preds, bs, h, w)        # :93-106
        self._last = dict(net=net, coords1=coords1, corr_block=corr_block)
        return [p for p in preds if p is not None] if last_only else preds

    def predict_bidirectional(self, inputs):
        """Flow in both directions of B image pairs, with forward-backward occlusion masks (an addition: tf-raft
        evaluates one direction).  inputs = [image1, image2], each (B, H, W, 3) float in 0..255 on the GPU.

        Returns (flow_fw, flow_bw, occ_fw, occ_bw): the finest (B, H, W, 2) flows image1 -> image2 and image2 -> image1
        after `iters_pred` iterations, what `predict_step` returns for [image1, image2] and for [image2, image1], and the
        torch.bool (B, H, W) masks of `fb_occlusion(flow_fw, flow_bw)` at its default thresholds.  Each image is encoded
        once by `fnet` and once by `cnet` (four image encodes where two calls make six), and both directions run as one
        loop at batch 2B with fmap1 = [f1; f2], fmap2 = [f2; f1].  Every image's result is independent of the batch it
        runs in, so on the native encoders (the f16x2 default) the flows equal the two single-direction calls bit for
        bit; the cuDNN encoders of the fp32 configuration may pick another algorithm for the other batch and differ in
        the last bits.  With `use_graph=True` the whole call, the occlusion check included, is captured once per input
        shape (apart from `__call__`'s graphs) and replayed; the returned tensors are then static buffers that the next
        call overwrites."""
        image1, image2 = inputs
        image1, image2 = _lib.f32c(image1), _lib.f32c(image2)
        if image1.shape != image2.shape:
            raise ValueError(f'image1 {tuple(image1.shape)} and image2 {tuple(image2.shape)} differ in shape')
        if self.iters_pred < 1:
            raise ValueError('predict_bidirectional needs iters_pred >= 1')
        self._sync_trained_params()
        if self.use_graph:
            return self._graph_run(('bidirectional', tuple(image1.shape)), self._bidirectional, (image1, image2))
        return self._bidirectional(image1, image2)

    def _bidirectional(self, image1, image2):
        bs, H, W, _ = image1.shape
        self._check_size(H, W)
        images = torch.cat([image1, image2])
        fmap = self.fnet(images, training=False, raw_image=True)                    # [f1; f2]
        net, inp = self._context(images, False)
        return self._iterate_bidirectional(fmap, torch.cat([fmap[bs:], fmap[:bs]]), net, inp, bs, H, W, None)

    def _iterate_bidirectional(self, fmap1, fmap2, net, inp, bs, H, W, flow_init):
        """Both directions of B pairs as one loop at batch 2B (first half a -> b, second half b -> a), then the occlusion
        check on the two halves of the finest prediction: (flow_fw, flow_bw, occ_fw, occ_bw)."""
        flow = self._iterate(fmap1, fmap2, net, inp, 2 * bs, H, W, False, True, flow_init)[-1]
        flow_fw, flow_bw = flow[:bs], flow[bs:]
        return (flow_fw, flow_bw) + fb_occlusion(flow_fw, flow_bw)

    def predict_video(self, frames, *, warm_start=True, bidirectional=False):
        """Flow along B video clips at once (an addition: tf-raft evaluates pairs only).

        `frames` is an iterable of (B, H, W, 3) CUDA tensors in 0..255, frame t of B independent clips.  A generator:
        for t = 1 .. T-1 it yields the finest (B, H, W, 2) flow from frame t-1 to frame t after `iters_pred`
        iterations, what `predict_step` returns for that pair.  Each frame is encoded by `fnet` once: its feature map
        serves as fmap2 of one pair and fmap1 of the next.  The feature encoder's instance norm works per image, so on
        the native encoders (the f16x2 default) the result does not depend on the batch the image was encoded in and
        every pair equals `__call__` bit for bit; the cuDNN encoders of the fp32 configuration may pick another
        algorithm for the smaller batch and differ in the last bits.  A step costs two image encodes (fnet on frame t,
        cnet on frame t-1) instead of the three of a `__call__` per pair.

        `warm_start=True`: from the second pair on, the loop starts from `forward_interpolate` of the previous pair's
        final low-resolution flow (coords1 - coords0), as RAFT does on Sintel and KITTI sequences; the first pair
        starts from zero flow.  `warm_start=False`: every pair starts from zero flow.

        `bidirectional=True`: it yields (flow_fw, flow_bw, occ_fw, occ_bw) for the pair (t-1, t), what
        `predict_bidirectional` returns for it.  `cnet` then runs once per frame too, and frame t's cached context
        serves the backward direction of pair (t-1, t) and the forward direction of pair (t, t+1), copied into the
        batch-2B loop (which writes it).  A step still costs two image encodes, fnet and cnet on frame t, and runs both
        directions as one loop at batch 2B.  The warm start extends RAFT's, which covers the forward direction only:
        the forward half starts from `forward_interpolate(F_low)` exactly as above, so the forward flows equal those of
        `bidirectional=False` bit for bit; the backward half starts from `-forward_interpolate(-B_low)`, B_low being
        the previous pair's backward low-resolution flow B_{t-1->t-2}.  Under constant velocity a point at x in frame
        t-1 with backward flow b was at x + b in frame t-2 and will be at x - b in frame t, so B_{t->t-1}(x - b) = b:
        splatting -b forward and negating the result gives it.  Both negations are exact.

        A frame whose shape differs from the first raises ValueError; fewer than two frames yield nothing.  Eager
        only: the video step is never captured into a CUDA graph, whatever `use_graph` says, and every yielded tensor
        is a new one."""
        self._sync_trained_params()
        if self.iters_pred < 1:
            raise ValueError('predict_video needs iters_pred >= 1')
        shape = coords0 = frame_prev = fmap_prev = flow_init = ctx_prev = None
        for t, frame in enumerate(frames):
            frame = _lib.f32c(frame)
            if shape is None:
                shape = tuple(frame.shape)
                if len(shape) != 4 or shape[-1] != 3:
                    raise ValueError(f'frames must be (B, H, W, 3); got {shape}')
                bs, H, W, _ = shape
                self._check_size(H, W)
            elif tuple(frame.shape) != shape:
                raise ValueError(f'frame {t}: shape {tuple(frame.shape)} differs from the first frame {shape}')
            fmap = self.fnet(frame, training=False, raw_image=True)                    # model.py:74, frame t only
            if bidirectional:
                ctx = self._context(frame, False)                                      # :82-86, frame t only
            if frame_prev is not None:
                if bidirectional:
                    net, inp = (torch.cat([p, c]) for p, c in zip(ctx_prev, ctx))     # copies: the loop writes net
                    out = self._iterate_bidirectional(torch.cat([fmap_prev, fmap]), torch.cat([fmap, fmap_prev]), net,
                                                      inp, bs, H, W, flow_init)
                else:
                    net, inp = self._context(frame_prev, False)                            # :82-86
                    out = self._iterate(fmap_prev, fmap, net, inp, bs, H, W, False, True, flow_init)[-1]
                if warm_start:
                    if coords0 is None:
                        coords0 = coords_grid(2 * bs if bidirectional else bs, H // 8, W // 8, self.device)
                    # flow_low = coords1 - coords0 with flow_advance_kernel's fp32 subtraction
                    if bidirectional:                           # [F_low; B_low] -> [fi(F_low); -fi(-B_low)], one launch
                        flow_low = self._last['coords1'] - coords0
                        flow_low[bs:].neg_()
                        flow_init = forward_interpolate(flow_low)
                        flow_init[bs:].neg_()
                    else:
                        flow_init = forward_interpolate(self._last['coords1'] - coords0)
                yield out
            frame_prev, fmap_prev = frame, fmap
            if bidirectional:
                ctx_prev = ctx

    call = __call__

    # -- keras-style steps (model.py:111-170) ---------------------------------------------------
    def compile(self, optimizer=None, clip_norm=None, loss=sequence_loss, epe=end_point_error, train_precision='fp32',
                **kwargs):
        """train_precision: 'fp32' (IEEE-fp32 library convolutions) or 'f16x2' (the training step's stride-1
        convolutions with cin >= 64 forward and backward on the tensor cores, fp16 hi/lo three-pass; DESIGN.md section 9)."""
        from .train import TRAIN_PRECISIONS
        if train_precision not in TRAIN_PRECISIONS:
            raise ValueError(f'unknown train_precision {train_precision!r}; expected one of {", ".join(TRAIN_PRECISIONS)}')
        self.train_precision = train_precision
        if self._trainer is not None:
            self._trainer.graph.train_precision = train_precision
        self.optimizer = optimizer
        self.clip_norm = clip_norm
        self.loss = loss
        self.epe = epe
        self.flow_metrics = OrderedDict((k, [0.0, 0]) for k in ('loss', 'epe', 'u1', 'u3', 'u5'))
        if self._pending_slots is not None and optimizer is not None:
            self._build_trainer()

    def fit(self, x, epochs=1, callbacks=None, steps_per_epoch=None, validation_data=None, validation_steps=None,
            verbose=1):
        """Keras's `Model.fit` as the reference's training scripts use it; see `tf_raft_b200.fit.fit`."""
        from .fit import fit
        return fit(self, x, epochs=epochs, callbacks=callbacks, steps_per_epoch=steps_per_epoch,
                   validation_data=validation_data, validation_steps=validation_steps, verbose=verbose)

    def _metric_update(self, key, value):
        m = self.flow_metrics[key]
        m[0] += float(value)
        m[1] += 1

    def _metric_results(self):
        return {k: (s / n if n else 0.0) for k, (s, n) in self.flow_metrics.items()}

    def train_step(self, data):
        """model.py:126-144: forward with training=True under autograd, sequence loss, clip_by_global_norm,
        optimizer.apply_gradients, metrics.  data = (image1, image2, flow_gt, valid) on the GPU.  With
        `compile(loss=UnsupervisedLoss())` the step is self-supervised: data = (image1, image2) or (image1, image2,
        flow_gt, valid), the bidirectional graph and that loss, epe / u1 / u3 / u5 of the forward final prediction when
        ground truth is given and not updated otherwise (tf_raft_b200/train.py).  Under an initialised
        torch.distributed process group the gradients are all-reduced (one flat NCCL call) and the context encoder's
        BatchNorm statistics are taken over the global batch (tf_raft_b200/train.py)."""
        from .train import AdamW
        if self.flow_metrics is None or getattr(self, 'optimizer', None) is None:
            raise RuntimeError('compile(optimizer=..., clip_norm=...) before train_step, as in train_chairs.py:92-98')
        if not isinstance(self.optimizer, AdamW):
            raise TypeError('optimizer must be tf_raft_b200.train.AdamW (tfa.optimizers.AdamW semantics)')
        if self._trainer is None:
            self._build_trainer()
        loss, info = self._trainer.step(data, self.optimizer, self.clip_norm, self.loss, self.epe)
        self._params_stale = True                      # the layers' own copies are refreshed on the next inference call
        self._metric_update('loss', loss)
        if info is not None:                           # UnsupervisedLoss on a batch without ground truth
            for k in ('epe', 'u1', 'u3', 'u5'):
                self._metric_update(k, info[k])
        return self._metric_results()

    def _sync_trained_params(self):
        if self._trainer is not None and self._params_stale:
            trainer = self._trainer
            self.load_params(trainer.params())         # copies into the layers, drops prepared blobs and graphs
            self._trainer = trainer
            self._params_stale = False

    def test_step(self, data):
        """model.py:146-159."""
        if self.flow_metrics is None:
            self.compile()
        image1, image2, flow, valid = data
        preds = self([image1, image2], training=False, last_only=True)
        info = self.epe([flow, valid], preds[-1])
        for k in ('epe', 'u1', 'u3', 'u5'):
            self._metric_update(k, info[k])
        return self._metric_results()

    def predict_step(self, data):
        """model.py:161-166: only the finest prediction."""
        image1, image2, *_ = data
        return self([image1, image2], training=False, last_only=True)[-1]

    def reset_metrics(self):
        if self.flow_metrics is not None:
            for m in self.flow_metrics.values():
                m[0], m[1] = 0.0, 0


class SmallRAFT(RAFT):
    _variant = _lib.VARIANT_SMALL

    def _build_layers(self, seed):
        self.hidden_dim = 96
        self.context_dim = 64
        self.corr_levels = 4
        self.corr_radius = 3
        s = 0 if seed is None else seed
        self.fnet = SmallEncoder(output_dim=128, norm_type='instance', drop_rate=self.drop_rate, device=self.device,
                                 seed=s, backend=self._encoder_backend())
        self.cnet = SmallEncoder(output_dim=self.hidden_dim + self.context_dim, norm_type=None,
                                 drop_rate=self.drop_rate, device=self.device, seed=s + 1, backend=self._encoder_backend())
        self.update_block = SmallUpdateBlock(filters=self.hidden_dim, precision=self.precision, device=self.device,
                                             seed=s + 2)

    def upsample_flow(self, flow, mask=None):
        """SmallRAFT upsamples with upflow8 (model.py:223)."""
        return upflow8(flow)
