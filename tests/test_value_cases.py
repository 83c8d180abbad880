"""CPU checks behind tests/test_gpu_values.py: known answers of the NumPy emulation of the fp16 hi/lo split, and the
fp64 oracle's NaN masks against a structural receptive-field propagation (cases.dilate).  The GPU tests compare the
kernels' NaN masks with the oracle's; these show that the oracle's masks are the receptive fields themselves, so that a
BLAS or convolution algorithm that spread NaN beyond them (or dropped one) could not pass for the reference."""
import numpy as np
import pytest
import torch

import cases
from oracle import raft_torch as rt, weights

F64 = torch.float64


def _bits16(x):
    return np.asarray(x, dtype=np.float16).view(np.uint16).tolist()


@pytest.mark.parametrize('v,hi,lo', [
    (1 + 2.0 ** -20, 1.0, 2.0 ** -20),            # lo subnormal in fp16 (2^-20 < 2^-14), exact
    (2.0 ** -25, 0.0, 0.0),                        # half the least fp16 subnormal: ties to even, lost
    (2.0 ** -30, 0.0, 0.0),                        # below fp16: lost
    (2.0 ** -24 * 3, 2.0 ** -24 * 3, 0.0),         # an fp16 subnormal: exact in hi
    (65504 + 100, 65504.0, 0.0),                   # beyond fp16: saturated
    (-65504 - 100, -65504.0, 0.0),
    (-0.0, -0.0, 0.0),                             # hi keeps the sign, lo = -0 - -0 = +0
])
def test_split_emulation_known_answers(v, hi, lo):
    h, l = cases.split_f16(np.array([v], dtype=np.float32))
    assert _bits16(h) == _bits16([hi]) and _bits16(l) == _bits16([lo]), (v, h, l)


def test_split_emulation_non_finite():
    h, l = cases.split_f16(np.array([np.nan, np.inf, -np.inf], dtype=np.float32))
    assert np.isnan(h[0]) and np.isnan(l[0])
    assert _bits16(h[1:]) == _bits16([65504, -65504]) and _bits16(l[1:]) == _bits16([0, 0])   # inf saturates too


def test_split_emulation_error_window():
    """hi + lo reproduces v to 2^-22 relative while lo is an fp16 normal (|v| >= 2^-3); below, the absolute error floors
    at half the least fp16 subnormal, 2^-25."""
    v = np.random.default_rng(0).uniform(1, 2, 4096).astype(np.float32)
    for e in (-20, -14, -8, -3, 0, 8, 14):
        x = v * np.float32(2.0 ** e)
        h, l = cases.split_f16(x)
        err = np.abs(h.astype(np.float64) + l - x.astype(np.float64))
        assert err.max() <= max(2.0 ** -22 * np.abs(x).max(), 2.0 ** -25), e


def _spatial(t):
    """(B, C, H, W) tensor -> (B, H, W) mask of the pixels that hold a NaN in any channel."""
    return torch.isnan(t).any(dim=1).numpy()


@pytest.mark.parametrize('size', [(70, 98), (36, 52)], ids=lambda s: 'x'.join(map(str, s)))
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_oracle_encoder_nan_mask_is_the_receptive_field(variant, size):
    """One NaN image pixel per image in a 3-image batch, at the corners and the middle (the stride-2 stages see odd
    sizes, so the asymmetric 'same' padding is traced)."""
    H, W = size
    p = cases.encoder_params(variant, None, 64, seed=5)
    im = np.random.default_rng(1).uniform(-1, 1, (3, H, W, 3)).astype(np.float32)
    pts = [(0, 0, 0, 0), (1, H - 1, W - 1, 2), (2, H // 2 + 1, W // 2 - 3, 1)]
    for b, y, x, c in pts:
        im[b, y, x, c] = np.nan
    got = _spatial(rt.encoder(rt.Ops(p, F64), torch.from_numpy(im).permute(0, 3, 1, 2).double(), 'enc', None, False))
    mask = np.zeros((3, H, W), dtype=bool)
    for b, y, x, _ in pts:
        mask[b, y, x] = True
    want = cases.encoder_field(mask)
    assert got.shape == want.shape and np.array_equal(got, want), (int(got.sum()), int(want.sum()))


@pytest.mark.parametrize('which', ['net', 'inp', 'corr', 'flow'])
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_oracle_update_block_nan_mask_is_the_receptive_field(variant, which):
    """One NaN in one input of the update block (image 1 of 2, the last channel): the NaN masks of net, delta and the
    mask head are the receptive field of that pixel through the motion encoder, the GRU and the heads."""
    b, h, w = 2, 13, 17
    ins = list(cases.update_inputs(variant, b, h, w, seed=3))
    k = ['net', 'inp', 'corr', 'flow'].index(which)
    y, x = 3, w - 2
    ins[k] = ins[k].copy()
    ins[k][1, y, x, -1] = np.nan
    p = weights.init_params(variant, 1234, bias_scale=0.05)
    fn = rt.basic_update_block if variant == 'raft' else rt.small_update_block
    net, mask, delta = fn(rt.Ops(p, F64), *[torch.from_numpy(a).permute(0, 3, 1, 2).double() for a in ins])
    masks = [np.zeros((b, h, w), dtype=bool) for _ in ins]
    masks[k][1, y, x] = True
    f_net, f_delta, f_mask = cases.update_field(variant, *masks)
    assert not f_net[0].any() and f_net[1].any()
    assert np.array_equal(_spatial(net), f_net)
    assert np.array_equal(_spatial(delta), f_delta)
    if mask is not None:
        assert np.array_equal(_spatial(mask), f_mask)
    # a NaN-free channel never turns NaN where the field says finite, and every channel is NaN where it says NaN
    assert np.array_equal(torch.isnan(net).all(dim=1).numpy(), f_net)
