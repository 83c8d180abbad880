"""Data-parallel self-supervised training on CPU, world_size 2 over gloo (127.0.0.1): with the batch sharded over the
ranks, UnsupervisedLoss normalises every rank's census sum by the mask count of the whole batch, so that averaging the
ranks' gradients reproduces the gradient of the whole batch (DESIGN.md sections 7 and 9.1).  The CUDA pieces (lookup,
correlation, census and occlusion) are replaced by the CPU stand-ins of test_unsup_ref.py, and the loss function by
the float64 oracle, which honours the census normalisers the loss hands it.

Both levels are discriminating: the two shards' mask counts differ by more than 5 %, and a per-shard normaliser (each
rank dividing by its own count) moves the averaged gradient far outside the tolerances."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

B, H, W, N = 2, 24, 40, 2
STEP_ALPHA = (0.0, 12.0)             # |F + g|^2 <= 12 px^2: about a third of a random-init RAFT's pixels consistent


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


class _CpuUnsupLossNorm:
    """train._UnsupLoss restated by the oracle in float64, census normalisers included: (2n, B, H, W, 2) flows,
    [image1; image2] census, images and occlusion, then the weights and optionally the (fw, bw) normalisers.  The loss
    comes back in the flows' dtype."""
    @staticmethod
    def apply(flows, census, images, occ, census_weight, smoothness_weight, edge_weight, gamma, census_norm=None):
        from oracle import unsup_np
        n, b = flows.shape[0] // 2, flows.shape[1]
        mask = torch.from_numpy(unsup_np.border_mask(2 * b, *flows.shape[2:4])) & ~occ
        norm = [None, None] if census_norm is None else [float(v) for v in census_norm]
        fw = unsup_np.direction_terms(census[:b], census[b:], images[:b], mask[:b], list(flows[:n]), gamma, edge_weight,
                                      norm[0])
        bw = unsup_np.direction_terms(census[b:], census[:b], images[b:], mask[b:], list(flows[n:]), gamma, edge_weight,
                                      norm[1])
        return (census_weight * (fw[0] + bw[0]) / 2 + smoothness_weight * (fw[1] + bw[1]) / 2).to(flows.dtype)


def _setup(rank, world, port):
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, here); sys.path.insert(0, os.path.dirname(here))
    import tf_raft_b200.losses as L
    import tf_raft_b200.train as tr
    from oracle import unsup_np
    from test_unsup_ref import _CpuCorrBlock, _CpuLookup, _cpu_occlusion
    from test_train_dist_unsup import _CpuUnsupLossNorm
    tr._Lookup, tr.CorrBlock, tr._UnsupLoss = _CpuLookup, _CpuCorrBlock, _CpuUnsupLossNorm
    L.census_transform = lambda im: torch.from_numpy(unsup_np.census(im.numpy()))
    L.fb_occlusion = _cpu_occlusion
    torch.set_num_threads(2)
    if world > 1:
        os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
        dist.init_process_group('gloo', rank=rank, world_size=world)


def _mask_counts(preds_fw, preds_bw, alpha):
    """(fw, bw) mask counts of the whole batch's images, one row per image."""
    from oracle import occlusion_np, unsup_np
    occ = occlusion_np.fb_occlusion(preds_fw[-1].detach().numpy(), preds_bw[-1].detach().numpy(), *alpha)
    border = unsup_np.border_mask(*occ[0].shape)
    return np.stack([(border & ~o).sum((1, 2)) for o in occ], 1)


def _loss_level(rank, world, q, port):
    """Given predictions (float64 leaves, image 0's much rougher than image 1's, so their occlusion differs), this
    rank's loss and its gradient with respect to every prediction of the whole batch (zero outside its shard); with
    world > 1 both summed over the ranks and divided by the world size."""
    _setup(rank, world, port)
    try:
        from test_gpu_unsup import _texture
        from tf_raft_b200 import UnsupervisedLoss
        im1, im2 = _texture(B, H, W, 1), _texture(B, H, W, 2)
        rng = np.random.default_rng(4)
        spread = np.array([4.0, 0.7])[:, None, None, None]
        preds = [torch.from_numpy(rng.standard_normal((B, H, W, 2)) * spread).requires_grad_(True) for _ in range(2 * N)]
        lo, hi = (rank, rank + 1) if world > 1 else (0, B)
        fw, bw = [p[lo:hi] for p in preds[:N]], [p[lo:hi] for p in preds[N:]]
        loss = UnsupervisedLoss()((torch.from_numpy(im1[lo:hi]), torch.from_numpy(im2[lo:hi])), (fw, bw))
        assert loss.dtype == torch.float64
        flat = torch.cat([g.flatten() for g in torch.autograd.grad(loss, preds)]).detach()
        loss = loss.detach().reshape(1)
        if world > 1:
            for t in (flat, loss):
                dist.all_reduce(t)
                t /= world
        counts = _mask_counts(preds[:N], preds[N:], (0.01, 0.5))
        out = (rank, flat.numpy(), float(loss), counts)
        if q is not None:
            q.put(out)
        return out
    finally:
        if world > 1:
            dist.destroy_process_group()


def _step_level(rank, world, q, port):
    """The flat gradient of RAFT's unsupervised step (forward_bidirectional on this rank's shard, UnsupervisedLoss with
    tight fb-consistency thresholds), all-reduced and divided by the world size as Trainer does, and cnet's moving
    statistics."""
    _setup(rank, world, port)
    try:
        import cases
        from oracle import weights
        import tf_raft_b200.train as tr
        from tf_raft_b200 import UnsupervisedLoss
        p = weights.init_params('raft', 21, bias_scale=0.05, norm_jitter=0.1)
        im1, im2 = cases.images(2, 64, 96, 3, 4)
        lo, hi = (rank, rank + 1) if world > 1 else (0, 2)
        frozen = ('moving_mean', 'moving_variance')
        P = {k: torch.tensor(v, dtype=torch.float32, requires_grad=not k.endswith(frozen)) for k, v in p.items()}
        names = [k for k, v in P.items() if v.requires_grad]
        moving = {k: v.detach().clone() for k, v in P.items() if k.endswith(frozen)}
        graph = tr.TrainGraph(P, 'raft', 'fp32', moving)
        t1, t2 = (torch.from_numpy(im[lo:hi]) for im in (im1, im2))
        preds = graph.forward_bidirectional(t1, t2, 2)
        loss = UnsupervisedLoss(alpha1=STEP_ALPHA[0], alpha2=STEP_ALPHA[1])((t1, t2), preds)
        g = torch.autograd.grad(loss, [P[k] for k in names])
        flat = torch.cat([x.flatten() for x in g])
        if world > 1:
            dist.all_reduce(flat)                     # the ONE flat gradient all-reduce of Trainer.step
            flat /= world
        mov = torch.cat([moving[k].flatten() for k in sorted(moving)])
        counts = _mask_counts(preds[0], preds[1], STEP_ALPHA)
        out = (rank, flat.numpy(), mov.numpy(), counts)
        if q is not None:
            q.put(out)
        return out
    finally:
        if world > 1:
            dist.destroy_process_group()


def _sharded(fn):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=fn, args=(r, 2, q, port)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=600) for _ in procs), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return res


def _assert_counts_differ(counts):
    """counts (B, 2): per image and direction; the shards are the images."""
    for d in range(2):
        a, b = sorted(int(c) for c in counts[:, d])
        assert a > 0 and b >= 1.05 * a, f'direction {d}: shard mask counts {a} and {b} differ by less than 5 %'


def test_sharded_unsupervised_loss_gradient_equals_the_whole_batch_world2_gloo():
    _, want, want_loss, counts = _loss_level(0, 1, None, 0)
    _assert_counts_differ(counts)
    scale = float(np.abs(want).max())
    for rank, got, loss, _ in _sharded(_loss_level):
        err = float(np.abs(got - want).max())
        assert err <= 1e-12 * scale, f'rank {rank}: gradient error {err:.3e} of {scale:.3e}'
        assert loss == pytest.approx(want_loss, rel=1e-12), f'rank {rank}: mean loss {loss!r}, whole batch {want_loss!r}'


def test_sharded_unsupervised_training_gradients_equal_the_whole_batch_world2_gloo():
    """The fp32 forwards of the whole batch and of a shard differ in the last bits, and a landing within that of a texel
    boundary takes the other bilinear corners (test_unsup_ref.py): at this seed that moves the flat gradient by 3.1e-3
    of its largest entry, so the bound is 1e-2.  Each rank dividing by its own mask count moves it by 1.6e-1."""
    want, want_mov, counts = _step_level(0, 1, None, 0)[1:]
    _assert_counts_differ(counts)
    scale = float(np.abs(want).max())
    for rank, got, mov, _ in _sharded(_step_level):
        err = float(np.abs(got - want).max())
        assert err <= 1e-2 * scale + 2e-6, f'rank {rank}: gradient error {err:.3e} of {scale:.3e}'
        np.testing.assert_allclose(mov, want_mov, atol=1e-6)      # moving statistics follow the GLOBAL 2B images
