"""The teacher-forced float64 training reference (oracle/teacher_forced.py) on the CPU: its float32 sampling positions
against the kernels' NumPy emulations bit for bit, its replay of recorded positions against the run that produced them,
and the oracle's float64 forward on the CPU after the device plumbing that lets it run on the GPU."""
import numpy as np
import pytest
import torch

import cases
from oracle import determinism_np as dnp, raft_pytorch as rp, raft_torch as rt, teacher_forced as tfo, weights

F32 = np.float32


def _coords(n, seed, lo, hi):
    rng = np.random.default_rng(seed)
    c = rng.uniform(lo, hi, (n, 2)).astype(F32)
    c[: n // 4] = np.round(c[: n // 4])                          # integers
    c[n // 4: n // 2] = np.round(c[n // 4: n // 2] * 8) / 8      # sums that land on integers at coarser levels
    return c


@pytest.mark.parametrize('n', [7, 62, 1000])
def test_tf_positions_equal_the_lookup_backward_emulation(n):
    """u = fl32(fl32(c * 2^-l) + (a - r)) per level and tap, as the clipped position g = floor + w0 and the clip gate of
    oracle/determinism_np (corr_lookup_bwd_kernel's arithmetic), bit for bit; coordinates inside, on and outside
    [0, n-1], integers and near-integers."""
    r = 4
    c = np.concatenate([_coords(4000, n, -12.0, n + 12.0),
                        np.array([[3 - 2 ** -22, 3 - 2 ** -22], [-2 ** -30, 2 ** -30], [n - 1, 0.5]], F32)])
    for level in range(4):
        u = tfo.tf_positions(torch.from_numpy(c), level, r).numpy()          # (Q, 2r+1, 2r+1, 2)
        inv = F32(1.0 / (1 << level))
        for a in range(2 * r + 1):
            X = dnp._axis(c[:, 0] * inv, a - r, n)
            ux = u[:, a, 0, 0]
            g = X['i0'].astype(F32) + X['w0']
            assert np.array_equal(np.clip(ux, 0, n - 1).view(np.uint32), g.view(np.uint32))
            assert np.array_equal((ux >= 0) & (ux <= n - 1), X['gate'])
        for b in range(2 * r + 1):
            Y = dnp._axis(c[:, 1] * inv, b - r, n)
            uy = u[:, 0, b, 1]
            g = Y['i0'].astype(F32) + Y['w0']
            assert np.array_equal(np.clip(uy, 0, n - 1).view(np.uint32), g.view(np.uint32))
        assert np.array_equal(u[:, :, :, 0], np.broadcast_to(u[:, :, :1, 0], u.shape[:3]))
        assert np.array_equal(u[:, :, :, 1], np.broadcast_to(u[:, :1, :, 1], u.shape[:3]))


def test_tf_positions_round_as_the_kernel_across_a_binade():
    """c = 3 - 2^-22 plus tap offset 4: the float32 sum crosses into [4, 8) and rounds to 7.0, an integer where the
    exact sum is not.  The kernel sees a zero-weight corner and a zero slope there; so must the reference."""
    c = torch.tensor([[3 - 2 ** -22, 1.5]], dtype=torch.float32)
    u = tfo.tf_positions(c, 0, 4)
    assert float(u[0, 8, 0, 0]) == 7.0                                   # tap a = 8: offset +4
    assert 3 - 2 ** -22 + 4 != 7.0
    X = dnp._axis(c[:, 0].numpy(), 4, 64)
    assert X['i0'][0] == X['i1'][0] == 7 and X['w0'][0] == 0 and X['w1'][0] == 0
    # the teacher-forced sampler there: tf-raft's floor / ceil sampler gives 0 at an integer position (both weights
    # 0) and no gradient; at the exact float64 position it would give ~7 and a slope of 1
    img = torch.arange(64.0, dtype=torch.float64).expand(64, 64).reshape(1, 64, 64, 1)     # the value at (x, y) is x
    cb = rt.CorrBlock.__new__(rt.CorrBlock)
    cb.corr_pyramid, cb.num_levels, cb.radius = [img], 1, 4
    x = c.double().reshape(1, 1, 1, 2).requires_grad_(True)
    tap = 8 * 9 + 4                                                      # x offset +4, y offset 0
    out = tfo.tf_retrieve(cb, x, c.reshape(1, 1, 1, 2))[0, 0, 0, tap]
    (g,) = torch.autograd.grad(out, x)
    assert float(out) == 0.0 and float(g[..., 0]) == 0.0
    free = rt.CorrBlock.retrieve(cb, x)[0, 0, 0, tap]
    (g,) = torch.autograd.grad(free, x)
    assert float(free) == pytest.approx(7 - 2 ** -22, abs=1e-9) and float(g[..., 0]) == pytest.approx(1.0)


@pytest.mark.parametrize('n', [5, 31, 62])
def test_grid_positions_equal_raft_pytorch_axis(n):
    """ATen's normalise / unnormalise in float32: weights and in-frame corners from grid_positions equal
    oracle/raft_pytorch._axis (the grid_sample lookup's emulation) bit for bit."""
    v = _coords(4000, n + 1, -6.0, n + 6.0).reshape(-1)
    v = np.concatenate([v, np.array([0, n - 1, -1, n, 2 ** 40, -2 ** 40], F32)])
    want = rp._axis(v, n)
    ix = tfo.grid_positions(torch.from_numpy(v), n).numpy()
    x0 = np.floor(ix)
    x1 = x0 + F32(1)
    got = (x1 - ix, ix - x0, np.where((x0 >= 0) & (x0 <= n - 1), x0, -1).astype(np.int64),
           np.where((x1 >= 0) & (x1 <= n - 1), x1, -1).astype(np.int64))
    for g, w in zip(got, want):
        assert np.array_equal(np.asarray(g).view(np.uint32) if g.dtype == F32 else g,
                              np.asarray(w).view(np.uint32) if w.dtype == F32 else w)


def test_grid_lookup_equals_raft_sampler_in_float64():
    """grid_lookup in float64 at the library's float32 grid_sample positions: within the float32 rounding of the
    weights of the library's lookup emulation (oracle/raft_pytorch.lookup_emulated), and within the float32 rounding of
    ATen's normalise / unnormalise of RAFT's F.grid_sample lookup (oracle/raft_pytorch.corr_lookup) in float64."""
    b, h, w = 1, 9, 13
    f1, f2 = cases.fmaps(b, h, w, 32, 5)
    pyr = rp.corr_pyramid(torch.from_numpy(f1).permute(0, 3, 1, 2).double(),
                          torch.from_numpy(f2).permute(0, 3, 1, 2).double())
    rng = np.random.default_rng(3)
    coords = (np.round(rng.uniform(-3, 16, (b, 2, h, w)) * 16) / 16).astype(F32)
    got = tfo.grid_lookup(pyr, torch.from_numpy(coords))
    emulated = rp.lookup_emulated([p[:, 0].float().numpy() for p in pyr], coords.transpose(0, 2, 3, 1), 4)
    scale = max(float(p.abs().max()) for p in pyr)
    err32 = float(np.abs(got.permute(0, 2, 3, 1).numpy() - emulated).max())
    err64 = float((got - rp.corr_lookup(pyr, torch.from_numpy(coords).double())).abs().max())
    print(f'grid_lookup: {err32:.2e} from the float32 emulation, {err64:.2e} from float64 F.grid_sample, '
          f'scale {scale:.2f}')
    assert err32 <= 4 * 2 ** -24 * scale
    assert err64 <= 64 * 2 ** -24 * scale


def _recording_retrieve(store, positions=None):
    """CorrBlock.retrieve that records its coordinates as float32; with positions='own', it samples at its own float32
    positions (teacher-forced by itself), else it is the plain sampler."""
    plain = rt.CorrBlock.retrieve

    def retrieve(self, coords):
        c32 = coords.detach().float()
        store.append(c32)
        return tfo.tf_retrieve(self, coords, c32) if positions == 'own' else plain(self, coords)
    return retrieve


def _run(params, data, variant, iters, dtype, retrieve=None, recorded=None):
    im1, im2, flow, valid = data
    if recorded is not None:
        loss, preds, grads, _ = tfo.tf_step(params, im1, im2, flow, valid, variant, recorded, dtype=dtype)
        return loss, grads
    leaves = {k: torch.as_tensor(v).to(dtype).requires_grad_(not k.endswith(tfo.FROZEN)) for k, v in params.items()}
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(rt.CorrBlock, 'retrieve', retrieve)
        preds = rt.forward(leaves, im1, im2, variant, iters, training=True, dtype=dtype)
    loss = tfo.sequence_loss(preds, flow, valid)
    names = [k for k, v in leaves.items() if v.requires_grad]
    return float(loss), dict(zip(names, torch.autograd.grad(loss, [leaves[k] for k in names])))


def _data(b, H, W):
    im1, im2 = cases.images(b, H, W, 3, 4)
    rng = np.random.default_rng(9)
    return im1, im2, (rng.standard_normal((b, H, W, 2)) * 3).astype(F32), rng.uniform(size=(b, H, W)) > 0.1


@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_teacher_forced_replay_equals_the_run_it_recorded(variant):
    """64x96, batch 1, 3 iterations.  A float64 run that samples at the float32 rounding of its own positions, under
    plain autograd, records them; tf_step replays the recording through `teacher_forced`.  Loss and every gradient
    agree to float64 rounding: the replay feeds iteration k the positions of iteration k and passes the coordinate
    gradient through unchanged."""
    iters = 3
    p = weights.init_params(variant, 21, bias_scale=0.05, norm_jitter=0.1)
    data = _data(1, 64, 96)
    rec = []
    loss_a, g_a = _run(p, data, variant, iters, torch.float64, _recording_retrieve(rec, 'own'))
    assert len(rec) == iters and all(r.dtype == torch.float32 for r in rec)
    loss_b, g_b = _run(p, data, variant, iters, torch.float64, recorded=rec)
    assert loss_b == pytest.approx(loss_a, rel=1e-13)
    for k, a in g_a.items():
        scale = float(a.abs().max()) + 1e-300
        assert float((g_b[k] - a).abs().max()) <= 1e-11 * scale, k


@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_teacher_forced_fp64_tracks_an_fp32_run(variant):
    """The reference fed the positions of an fp32 run (plain autograd, the oracle in float32) stays within fp32 error
    of that run's loss and whole gradient: the only differences left are rounding, none from sampling corners."""
    iters = 3
    p = weights.init_params(variant, 21, bias_scale=0.05, norm_jitter=0.1)
    data = _data(1, 64, 96)
    rec = []
    loss32, g32 = _run(p, data, variant, iters, torch.float32, _recording_retrieve(rec))
    loss64, g64 = _run(p, data, variant, iters, torch.float64, recorded=rec)
    num = sum(float(((g32[k].double() - g64[k]) ** 2).sum()) for k in g64)
    den = sum(float((g64[k] ** 2).sum()) for k in g64)
    print(f'{variant}: loss {abs(loss32 - loss64) / loss64:.2e} relative, '
          f'gradient {np.sqrt(num / den):.2e} relative L2')
    assert abs(loss32 - loss64) <= 1e-5 * loss64
    assert np.sqrt(num / den) <= 1e-3


def test_cpu_float64_forward_unchanged_by_device_plumbing():
    """oracle.raft_torch.forward(dtype=float64) on CPU inputs: CPU outputs, bit-identical to the forward with the
    aranges created without a device."""
    p = weights.init_params('raft', 3, bias_scale=0.05, norm_jitter=0.1)
    im1, im2 = cases.images(1, 64, 96, 5, 6)
    got = rt.forward(p, im1, im2, 'raft', 2, dtype=torch.float64)

    def coords_grid(batch_size, height, width, dtype=torch.float32, device=None):
        gy, gx = torch.meshgrid(torch.arange(height, dtype=dtype), torch.arange(width, dtype=dtype), indexing='ij')
        return torch.stack([gx, gy], dim=-1)[None].repeat(batch_size, 1, 1, 1)

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(rt, 'coords_grid', coords_grid)
        want = rt.forward(p, im1, im2, 'raft', 2, dtype=torch.float64)
    for g, w in zip(got, want):
        assert g.device.type == 'cpu' and g.dtype == torch.float64
        assert torch.equal(g, w)
