"""The original PyTorch RAFT's checkpoints on the CPU: the loader (`load_pytorch_checkpoint`) against synthetic
checkpoints in PyTorch layout, the mask head's channel permutation, the PyTorch-layout oracle's lookup, and a check
that the two conventions really differ at the sizes the GPU tests use.  No GPU needed."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import raft_pytorch as rp, raft_torch as rt, weights
from tf_raft_b200.checkpoint import load_pytorch_checkpoint, mask_head_permutation

EXPECT = weights.param_shapes('raft')


@pytest.fixture(scope='module')
def ckpt():
    return rp.synthetic_checkpoint(seed=3)


def _expect():
    return {k: np.zeros(s, np.float32) for k, s in EXPECT.items()}


def test_round_trip_through_a_file(ckpt, tmp_path):
    path = tmp_path / 'raft-synthetic.pth'
    torch.save(ckpt, path)
    params = load_pytorch_checkpoint(str(path), expect=_expect())
    assert set(params) == set(EXPECT)
    for k, v in params.items():
        assert v.dtype == np.float32 and v.shape == EXPECT[k], k
    sd = {k[len('module.'):]: v.numpy() for k, v in ckpt.items()}
    np.testing.assert_array_equal(params['fnet.conv1.kernel'], sd['fnet.conv1.weight'].transpose(2, 3, 1, 0))
    np.testing.assert_array_equal(params['update_block.gru.convz1.kernel'],
                                  sd['update_block.gru.convz1.weight'].transpose(2, 3, 1, 0))
    np.testing.assert_array_equal(params['cnet.layer2.0.downsample.1.moving_variance'],
                                  sd['cnet.layer2.0.norm3.running_var'])
    np.testing.assert_array_equal(params['cnet.norm1.gamma'], sd['cnet.norm1.weight'])
    np.testing.assert_array_equal(params['cnet.norm1.beta'], sd['cnet.norm1.bias'])
    np.testing.assert_array_equal(params['cnet.norm1.moving_mean'], sd['cnet.norm1.running_mean'])
    for k in ('fnet.norm1', 'fnet.layer3.1.norm2', 'fnet.layer2.0.downsample.1'):
        np.testing.assert_array_equal(params[k + '.gamma'], 1.0)
        np.testing.assert_array_equal(params[k + '.beta'], 0.0)
    perm = mask_head_permutation()
    np.testing.assert_array_equal(params['update_block.mask.2.kernel'][0, 0], sd['update_block.mask.2.weight'][perm, :, 0, 0].T)
    np.testing.assert_array_equal(params['update_block.mask.2.bias'], sd['update_block.mask.2.bias'][perm])
    # the same from the state dict itself, and without the DataParallel prefix
    plain = {k[len('module.'):]: v for k, v in ckpt.items()}
    again = load_pytorch_checkpoint(plain, expect=_expect())
    assert all(np.array_equal(again[k], params[k]) for k in params)


def test_mask_head_permutation_is_a_permutation():
    perm = mask_head_permutation()
    assert sorted(perm) == list(range(576))
    # channel (8a + b) * 9 + k here is k * 64 + 8a + b in RAFT's view(N, 1, 9, 8, 8, H, W)
    assert perm[(8 * 2 + 5) * 9 + 7] == 7 * 64 + 8 * 2 + 5


def test_error_paths(ckpt):
    plain = {k[len('module.'):]: v for k, v in ckpt.items()}

    def err(sd, **kw):
        with pytest.raises(ValueError) as e:
            load_pytorch_checkpoint(sd, expect=_expect(), **kw)
        return str(e.value)

    sd = dict(plain)
    del sd['update_block.flow_head.conv2.bias']
    assert 'missing' in err(sd) and 'update_block.flow_head.conv2.bias' in err(sd)
    sd = dict(plain)
    sd['update_block.extra.weight'] = torch.zeros(3, 3, 1, 1)
    assert 'unexpected' in err(sd) and 'update_block.extra.kernel' in err(sd)
    sd = dict(plain)
    sd['fnet.conv2.weight'] = torch.zeros(128, 128, 1, 1)
    assert 'shapes' in err(sd) and 'fnet.conv2.kernel' in err(sd)
    sd = dict(plain)
    sd['cnet.layer3.0.norm3.running_mean'] = sd['cnet.layer3.0.norm3.running_mean'] + 1
    assert 'norm3' in err(sd) and 'cnet.layer3.0.norm3.running_mean' in err(sd)
    sd = dict(plain)
    sd['fnet.layer1.0.conv3.weight'] = torch.zeros(64, 16, 1, 1)
    sd['fnet.layer1.0.norm4.weight'] = torch.zeros(64)
    assert 'RAFT-small' in err(sd)
    sd = dict(plain)
    sd['update_block.odd'] = torch.zeros(3)
    assert 'update_block.odd' in err(sd)
    with pytest.raises(ValueError, match='no fnet'):
        load_pytorch_checkpoint({'other.weight': torch.zeros(2, 2, 1, 1)})


def test_mask_permutation_upsamples_the_same():
    """tf-raft-layout convex upsampling with the permuted mask head equals RAFT's own upsampling with the original."""
    rng = np.random.default_rng(5)
    n, h, w = 2, 5, 7
    hid = torch.from_numpy(rng.standard_normal((n, 256, h, w)))
    wt = torch.from_numpy(rng.standard_normal((576, 256, 1, 1)) * 0.05)
    bias = torch.from_numpy(rng.standard_normal(576) * 0.1)
    flow = torch.from_numpy(rng.standard_normal((n, 2, h, w)) * 3)
    want = rp.upsample_flow(flow, F.conv2d(hid, wt, bias))                          # (n, 2, 8h, 8w)
    perm = torch.from_numpy(mask_head_permutation())
    mask_tf = F.conv2d(hid, wt[perm], bias[perm]).permute(0, 2, 3, 1)
    got = rt.upsample_flow(flow.permute(0, 2, 3, 1), mask_tf)                       # (n, 8h, 8w, 2)
    np.testing.assert_allclose(got.numpy(), want.permute(0, 2, 3, 1).numpy(), rtol=0, atol=1e-12)


@pytest.mark.parametrize('grid', [(2, 9, 13), (1, 8, 32), (2, 8, 9)])
def test_oracle_lookup_matches_grid_sample_and_the_emulation(grid):
    """The oracle's lookup is F.grid_sample; the float32 emulation of the kernel's order agrees with it in fp32 and with
    fp64, also on levels of height or width 1 (every tap 0) and far outside."""
    b, h, w = grid
    rng = np.random.default_rng(11)
    pyr64 = rp.corr_pyramid(torch.from_numpy(rng.standard_normal((b, 16, h, w))),
                            torch.from_numpy(rng.standard_normal((b, 16, h, w))))
    gy, gx = np.meshgrid(np.arange(h), np.arange(w), indexing='ij')
    coords = np.stack([gx, gy], -1)[None].repeat(b, 0) + rng.uniform(-6, 6, (b, h, w, 2))
    coords.reshape(-1, 2)[::5] = np.round(coords.reshape(-1, 2)[::5])
    coords.reshape(-1, 2)[1::9] += 1e3
    coords = coords.astype(np.float32)
    pyr32 = [p.float() for p in pyr64]
    want64 = rp.corr_lookup(pyr64, torch.from_numpy(coords).double().permute(0, 3, 1, 2)).permute(0, 2, 3, 1).numpy()
    want32 = rp.corr_lookup(pyr32, torch.from_numpy(coords).permute(0, 3, 1, 2)).permute(0, 2, 3, 1).numpy()
    emu = rp.lookup_emulated([p[:, 0].numpy() for p in pyr32], coords, 4)
    # torch's CPU divide rounds x / (S-1) directly where the CUDA kernel multiplies by the reciprocal: ix may differ in
    # its last bit, which moves a weight by up to ulp(ix) ~ 2^-23 * max(h, w)
    vmax = max(float(p.abs().max()) for p in pyr32)
    np.testing.assert_allclose(emu, want32, rtol=0, atol=2.0 ** -21 * max(h, w) * vmax)
    np.testing.assert_allclose(emu, want64, rtol=0, atol=1e-5 * max(1.0, np.abs(want64).max()))
    for l, p in enumerate(pyr32):
        if min(p.shape[2:]) == 1:
            assert not emu[..., l * 81:(l + 1) * 81].any(), f'level {l} {tuple(p.shape[2:])} must be all zero'


def test_emulation_nan_inf_and_huge_coordinates():
    img = np.arange(1, 1 + 6 * 7, dtype=np.float32).reshape(1, 6, 7)
    pyr = [img]
    for c in ([np.nan, 2.0], [np.inf, 2.0], [-np.inf, 2.0], [1e30, 2.0], [3.0, -1e30]):
        out = rp.lookup_emulated(pyr, np.array(c, np.float32).reshape(1, 1, 1, 2), 1)
        assert np.array_equal(out, np.zeros_like(out)), c
    # a NaN texel reaches the taps with that corner in frame, weight 0 included: tap (x 2, y 2) has x corners 2 and 3
    img2 = img.copy()
    img2[0, 2, 3] = np.nan
    out = rp.lookup_emulated([img2], np.array([3.0, 2.0], np.float32).reshape(1, 1, 1, 2), 1).reshape(3, 3)
    assert np.isnan(out[1, 1]) and np.isnan(out[0, 1]) and not np.isnan(out[2, 2])


def test_gpu_encoder_grids_cover_every_stride2_tile():
    """The GPU encoder test's sizes put a stride-2 convolution, which under PyTorch's padding starts its TMA box at an
    odd negative coordinate, on every (tile, input parity) pair, and include even sizes."""
    import ast
    import os
    import cases
    src = open(os.path.join(os.path.dirname(__file__), 'test_gpu_pytorch_conventions.py')).read()
    extra = next(ast.literal_eval(n.value.right) for n in ast.walk(ast.parse(src))
                 if isinstance(n, ast.Assign) and getattr(n.targets[0], 'id', '') == 'ENC_GRIDS')
    grids = list(cases.ENCODER_GRIDS) + list(extra)
    universe = {(tw, 128 // tw, oh, ow) for tw in (128, 64, 32, 16, 8) for oh in (0, 1) for ow in (0, 1)}
    assert set().union(*(cases.stride2_combos(H, W, 'raft') for H, W in grids)) == universe
    assert any(H % 16 == 0 and W % 16 == 0 for H, W in grids)


def test_conventions_differ_at_even_sizes(ckpt):
    """Non-vacuity: at even sizes the padding rules differ, and the two oracles' flows on the same weights differ."""
    for n in (64, 448, 512, 440, 1024):
        pt = rt._same_pads(n, 7, 2)[0]
        assert pt == 2, n                                  # Keras: 2 before at 7x7/s2 on even input; PyTorch: 3
        assert rt._same_pads(n // 2, 3, 2)[0] == 0         # Keras: 0 before at 3x3/s2; PyTorch: 1
    params = load_pytorch_checkpoint(ckpt, expect=_expect())
    im1 = np.random.default_rng(0).uniform(0, 255, (1, 64, 64, 3)).astype(np.float32)
    im2 = np.roll(im1, 3, axis=2)
    a = rp.forward(ckpt, im1, im2, iters=2)[0][-1]
    b = rt.forward(params, im1, im2, 'raft', 2, dtype=torch.float64)[-1]
    b = b.numpy() if isinstance(b, torch.Tensor) else b
    assert np.abs(a - b).max() > 1e-2
