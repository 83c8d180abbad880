"""Teacher-forced, stage-by-stage parity at the benchmark resolution (448x512, one pair).

Each CUDA stage is fed the ORACLE's inputs for that stage (not the GPU's own previous outputs), so an
error is attributed to the stage that makes it and recurrent amplification cannot hide or inflate it.
"""
import numpy as np
import pytest
import torch

import cases
from oracle import raft_torch as rt, weights

pytestmark = pytest.mark.gpu
ITERS = 12


def dev(a):
    if isinstance(a, torch.Tensor):
        return a.contiguous().cuda()
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def maxabs(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max())


@pytest.fixture(scope='module')
def oracle_run():
    p = weights.init_params('raft', 1234)
    im1, im2 = cases.images(1, 448, 512)
    preds, inter = rt.forward(p, im1, im2, 'raft', ITERS, return_intermediates=True)
    return p, im1, im2, preds, inter


@pytest.fixture(scope='module')
def T():
    import tf_raft_b200
    return tf_raft_b200


def test_encoders_are_fp32_grade(T, oracle_run):
    """RAFT's encoders as the model runs them under the default precision (f16x2: the native tensor-core encoders)
    against the fp32 oracle at 448x512, one pair, with zero biases and unit norm parameters.  tests/test_gpu_encoders.py
    compares the native encoders with the fp64 oracle at every stride-2 geometry and at the production batches."""
    p, im1, im2, _, inter = oracle_run
    model = T.RAFT(iters=ITERS, iters_pred=ITERS)
    model.load_params(p)
    fmap1, fmap2, net, inp = model._encode(dev(im1), dev(im2), False)
    errs = dict(fmap1=maxabs(fmap1, inter['fmap1']), fmap2=maxabs(fmap2, inter['fmap2']),
                net=maxabs(net, inter['net0']), inp=maxabs(inp, inter['inp']))
    print('encoder max-abs vs oracle:', errs, 'fmap magnitude', float(inter['fmap1'].abs().max()))
    assert max(errs.values()) < 2e-4, errs


@pytest.mark.parametrize('precision', ['f16x2', 'fp32'])
def test_pyramid_from_oracle_fmaps(T, oracle_run, precision):
    _, _, _, _, inter = oracle_run
    cb = T.CorrBlock(dev(inter['fmap1']), dev(inter['fmap2']), 4, 4, precision=precision)
    for l in range(4):
        want = inter['corr_pyramid'][l]
        e = maxabs(cb.corr_pyramid[l], want)
        print(f'{precision} pyramid level {l}: max-abs {e:.3e} (magnitude {float(want.abs().max()):.2f})')
        assert e < 1e-4


def test_lookup_bit_exact_every_iteration(T, oracle_run):
    """With the oracle's pyramid and the oracle's coordinates, the lookup is bit-identical at every iteration
    (includes iteration 0 where every level-0 tap is exactly 0, and coordinates far outside the image)."""
    _, _, _, _, inter = oracle_run
    cb = T.CorrBlock(dev(inter['fmap1']), dev(inter['fmap2']), 4, 4, precision='fp32')
    cb.corr_pyramid = [dev(q) for q in inter['corr_pyramid']]
    grid = rt.coords_grid(1, 56, 64)
    for i in (0, 1, 5, 11):
        coords = grid if i == 0 else inter['coords'][i - 1]
        got = cb.retrieve(dev(coords)).cpu()
        assert torch.equal(got, inter['corr'][i]), f'iteration {i}: {maxabs(got, inter["corr"][i])}'


@pytest.mark.parametrize('precision', ['f16x2', 'fp32'])
def test_update_block_teacher_forced(T, oracle_run, precision):
    p, _, _, _, inter = oracle_run
    blk = T.BasicUpdateBlock(precision=precision)
    blk.load_params(p, 'update_block.')
    grid = rt.coords_grid(1, 56, 64)
    for i in (0, 1, 6, 11):
        net_in = inter['net0'] if i == 0 else inter['net'][i - 1]
        coords = grid if i == 0 else inter['coords'][i - 1]
        flow = coords - grid
        n2, mask, delta = blk([dev(net_in), dev(inter['inp']), dev(inter['corr'][i]), dev(flow)])
        e = dict(net=maxabs(n2, inter['net'][i]), mask=maxabs(mask, inter['mask'][i]),
                 delta=maxabs(delta, inter['delta'][i]))
        print(f'{precision} update block, iteration {i}: max-abs {e}, |delta| up to '
              f'{float(inter["delta"][i].abs().max()):.2f}')
        assert e['net'] < 5e-5 and e['mask'] < 2e-4 and e['delta'] < 2e-4, (i, e)


def test_upsample_teacher_forced(T, oracle_run):
    _, _, _, preds, inter = oracle_run
    model = T.RAFT(iters=1, iters_pred=1)
    grid = rt.coords_grid(1, 56, 64)
    for i in (0, 11):
        flow = inter['coords'][i] - grid
        up = model.upsample_flow(dev(flow), dev(inter['mask'][i]))
        e = maxabs(up, preds[i])
        print(f'upsample iteration {i}: max-abs {e:.3e}')
        assert e < 1e-4


@pytest.mark.parametrize('variant,which', [('raft', 'fnet'), ('raft', 'cnet'), ('small', 'fnet'), ('small', 'cnet')])
def test_native_encoder_vs_oracle_and_cudnn(T, variant, which):
    """Tensor-core encoders (stride-2 TMA boxes, fused / reduced norms) against the oracle and against the
    IEEE-fp32 cuDNN restatement, with jittered norm parameters and non-zero biases, on a ragged 72x104 image."""
    from tf_raft_b200.layers.extractor import BasicEncoder, SmallEncoder
    p = weights.init_params(variant, 99, bias_scale=0.05, norm_jitter=0.2)
    cfg = rt.VARIANTS[variant]
    norm = cfg['fnorm'] if which == 'fnet' else cfg['cnorm']
    out_dim = {('raft', 'fnet'): 256, ('raft', 'cnet'): 256, ('small', 'fnet'): 128, ('small', 'cnet'): 160}[(variant, which)]
    cls = BasicEncoder if variant == 'raft' else SmallEncoder
    im1, _ = cases.images(3, 72, 104, seed0=5)
    x = 2 * (torch.from_numpy(im1) / 255.0) - 1.0
    ops = rt.Ops(p)
    want = rt.encoder(ops, x.permute(0, 3, 1, 2), which, norm, False).permute(0, 2, 3, 1)
    outs = {}
    for backend in ('native', 'torch'):
        enc = cls(output_dim=out_dim, norm_type=norm, backend=backend)
        enc.load_params(p, which + '.')
        outs[backend] = enc(dev(im1), training=False, raw_image=True)
        assert tuple(outs[backend].shape) == tuple(want.shape)
    e_nat, e_cud = maxabs(outs['native'], want), maxabs(outs['torch'], want)
    print(f'{variant}.{which} ({norm}): native max-abs {e_nat:.3e}, cuDNN-ieee max-abs {e_cud:.3e}, '
          f'|out| up to {float(want.abs().max()):.2f}')
    assert e_cud < 1e-4 and e_nat < 2e-4
    # normalised input path (the encoder layer on its own, as the reference calls it)
    enc = cls(output_dim=out_dim, norm_type=norm, backend='native')
    enc.load_params(p, which + '.')
    assert maxabs(enc(dev(x.numpy()), training=False), want) < 2e-4


def test_native_encoder_training_mode_batch_stats(T):
    """cnet BatchNorm with training=True uses batch statistics (extractor.py:10, keras semantics)."""
    from tf_raft_b200.layers.extractor import BasicEncoder
    p = weights.init_params('raft', 98, bias_scale=0.05, norm_jitter=0.2)
    im1, _ = cases.images(2, 64, 96, seed0=6)
    x = 2 * (torch.from_numpy(im1) / 255.0) - 1.0
    want = rt.encoder(rt.Ops(p), x.permute(0, 3, 1, 2), 'cnet', 'batch', True).permute(0, 2, 3, 1)
    enc = BasicEncoder(output_dim=256, norm_type='batch', backend='native')
    enc.load_params(p, 'cnet.')
    got = enc(dev(im1), training=True, raw_image=True)
    e = maxabs(got, want)
    print(f'cnet training-mode max-abs {e:.3e}')
    assert e < 2e-4
