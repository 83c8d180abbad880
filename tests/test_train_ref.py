"""The float64 restatement of the optimiser state (oracle/train_ref.py) on known answers, and the BatchNorm moving
statistics of the backward-capable training graph against it.  CPU only."""
import math

import numpy as np
import pytest
import torch

import cases
from oracle import raft_torch as rt, train_ref, weights

B1, B2, EPS = 0.9, 0.999, 1e-7


# --------------------------------------------------------------------------------------------- AdamW, worked by hand
def test_adamw_three_scalar_steps_worked_by_hand():
    """One variable p0 = 1, gradients 0.5, -0.25, 1.0, lr 0.1, wd 0.01, no clip.  The numbers below are the hand-worked
    moments; the step uses lr_t = lr sqrt(1 - b2^t) / (1 - b1^t) and the decay is not scaled by lr."""
    opt = train_ref.AdamW(0.01, 0.1)
    p = {'w': np.array([1.0])}
    # t = 1: m = 0.1 * 0.5, v = 0.001 * 0.25
    p = opt.apply(p, {'w': np.array([0.5])})
    m1, v1 = 0.05, 0.00025
    p1 = 0.99 - 0.1 * math.sqrt(0.001) / 0.1 * m1 / (math.sqrt(v1) + EPS)
    assert opt.m['w'][0] == pytest.approx(m1, rel=1e-14) and opt.v['w'][0] == pytest.approx(v1, rel=1e-14)
    assert p['w'][0] == pytest.approx(p1, rel=1e-14)
    assert p1 == pytest.approx(0.89, abs=1e-6)          # t = 1: a step of lr * sign(g), up to epsilon
    # t = 2: m = 0.9 * 0.05 + 0.1 * -0.25 = 0.02, v = 0.999 * 0.00025 + 0.001 * 0.0625 = 0.00031225
    p = opt.apply(p, {'w': np.array([-0.25])})
    m2, v2 = 0.02, 0.00031225
    p2 = 0.99 * p1 - 0.1 * math.sqrt(0.001999) / 0.19 * m2 / (math.sqrt(v2) + EPS)
    assert opt.m['w'][0] == pytest.approx(m2, rel=1e-13) and opt.v['w'][0] == pytest.approx(v2, rel=1e-13)
    assert p['w'][0] == pytest.approx(p2, rel=1e-13)
    # t = 3: m = 0.9 * 0.02 + 0.1 * 1 = 0.118, v = 0.999 * 0.00031225 + 0.001 = 0.00131193775
    p = opt.apply(p, {'w': np.array([1.0])})
    m3, v3 = 0.118, 0.00131193775
    p3 = 0.99 * p2 - 0.1 * math.sqrt(0.002997001) / 0.271 * m3 / (math.sqrt(v3) + EPS)
    assert opt.m['w'][0] == pytest.approx(m3, rel=1e-13) and opt.v['w'][0] == pytest.approx(v3, rel=1e-13)
    assert p['w'][0] == pytest.approx(p3, rel=1e-13)
    assert opt.iterations == 3


def test_adamw_zero_gradient_only_decays():
    """A zero gradient leaves m and v at 0 and the Adam term at 0 / (0 + eps) = 0: only the decay moves the weight."""
    opt = train_ref.AdamW(0.05, 1e-3)
    p = {'w': np.array([2.0, -0.5, 0.0])}
    for _ in range(3):
        p = opt.apply(p, {'w': np.zeros(3)})
    np.testing.assert_allclose(p['w'], np.array([2.0, -0.5, 0.0]) * 0.95 ** 3, rtol=1e-15, atol=0)
    assert not opt.m['w'].any() and not opt.v['w'].any()


@pytest.mark.parametrize('clip_norm,scale', [(1.0, 0.2), (10.0, 1.0), (5.0, 1.0), (None, 1.0), (0.0, 1.0)],
                         ids=['active', 'inactive', 'at-the-norm', 'none', 'zero'])
def test_clip_by_global_norm(clip_norm, scale):
    """Two variables (3, 0) and (4): global norm 5.  The clip multiplies every gradient by clip / max(5, clip); None and
    0 disable it.  The clipped gradient is what m sees: m = (1 - b1) * scale * g after one step."""
    grads = {'a': np.array([3.0, 0.0]), 'b': np.array([4.0])}
    assert train_ref.global_sumsq(grads) == 25.0
    assert train_ref.clip_scale(25.0, clip_norm) == pytest.approx(scale, rel=1e-15)
    opt = train_ref.AdamW(0.0, 1e-3)
    opt.apply({'a': np.zeros(2), 'b': np.zeros(1)}, grads, clip_norm)
    np.testing.assert_allclose(opt.m['a'], (1 - B1) * scale * grads['a'], rtol=1e-15)
    np.testing.assert_allclose(opt.v['b'], (1 - B2) * (scale * 4.0) ** 2, rtol=1e-15)


# --------------------------------------------------------------------------------------------- schedule
def test_schedule_crosses_its_first_cycle_inside_adamw():
    """CyclicalLearningRate(1e-3, 2e-3, step_size 3, first_cycle_scaler): up over steps 0..3, down over 3..6, then the
    minimum for good (cycle 2 is scaled by 0).  AdamW evaluates it at `iterations` before the increment, and corrects the
    bias with t = iterations + 1."""
    from tf_raft_b200.train import CyclicalLearningRate, first_cycle_scaler
    want = [1e-3, 4e-3 / 3, 5e-3 / 3, 2e-3, 5e-3 / 3, 4e-3 / 3, 1e-3, 1e-3, 1e-3, 1e-3]

    def sched(s):
        return train_ref.cyclical_lr(s, 1e-3, 2e-3, 3, first_cycle_scaler)
    np.testing.assert_allclose([sched(s) for s in range(10)], want, rtol=1e-14)
    project = CyclicalLearningRate(1e-3, 2e-3, step_size=3, scale_fn=first_cycle_scaler)
    np.testing.assert_allclose([project(s) for s in range(40)], [sched(s) for s in range(40)], rtol=1e-15)
    opt = train_ref.AdamW(0.0, sched)
    p = {'w': np.zeros(1)}
    for s in range(8):
        t = s + 1
        assert opt.lr() == pytest.approx(want[s], rel=1e-14)
        assert opt.lr_t() == pytest.approx(want[s] * math.sqrt(1 - B2 ** t) / (1 - B1 ** t), rel=1e-14)
        p = opt.apply(p, {'w': np.ones(1)})


# --------------------------------------------------------------------------------------------- BatchNorm moving statistics
def test_bn_moving_update_known_answer():
    """Batch mean 1, biased variance 2 over n = 4 values: the moving variance takes 2 * 4/3, the mean as it is."""
    moving = {'x.moving_mean': np.array([0.5]), 'x.moving_variance': np.array([1.0])}
    out = train_ref.bn_moving_update(moving, {'x': (np.array([1.0]), np.array([2.0]), 4)})
    assert out['x.moving_mean'][0] == pytest.approx(0.99 * 0.5 + 0.01 * 1.0, rel=1e-15)
    assert out['x.moving_variance'][0] == pytest.approx(0.99 * 1.0 + 0.01 * 8.0 / 3.0, rel=1e-15)


def test_oracle_bn_record_leaves_outputs_unchanged():
    """Recording the batch statistics does not change what the oracle encoder computes, and it records every BatchNorm
    layer of the context encoder with its per-channel count."""
    p = weights.init_params('raft', 21, bias_scale=0.05, norm_jitter=0.1)
    im, _ = cases.images(2, 32, 48, 7, 8)
    x = torch.from_numpy(2 * (im / 255.0) - 1.0).permute(0, 3, 1, 2)
    rec = {}
    plain = rt.encoder(rt.Ops(p), x, 'cnet', 'batch', True)
    recorded = rt.encoder(rt.Ops(p, bn_record=rec), x, 'cnet', 'batch', True)
    assert torch.equal(plain, recorded)
    layers = sorted(k[:-len('.moving_mean')] for k in p if k.startswith('cnet.') and k.endswith('.moving_mean'))
    assert sorted(rec) == layers and len(layers) == 15
    assert rec['cnet.norm1'][2] == 2 * 16 * 24 and rec['cnet.layer3.1.norm2'][2] == 2 * 4 * 6


def _graph_moving_after(passes, P, moving):
    import tf_raft_b200.train as tr
    graph = tr.TrainGraph(P, 'raft', 'fp32', moving)
    for im in passes:
        with torch.no_grad():
            graph.encoder(torch.from_numpy(2 * (im / 255.0) - 1.0).permute(0, 3, 1, 2).float(), 'cnet', 'batch')
    return moving


@pytest.mark.parametrize('npasses', [1, 3])
def test_train_graph_moving_statistics_follow_keras(npasses):
    """TrainGraph's context encoder in training mode at 32x48, batch 2 (n from 2*16*24 = 768 down to 2*4*6 = 48 values
    per channel, a Bessel factor up to 48/47): after each forward the moving statistics equal the restatement advanced by
    the fp64 oracle's own batch statistics, to fp32 rounding -- and they do not equal the biased-variance rule."""
    p = weights.init_params('raft', 21, bias_scale=0.05, norm_jitter=0.1)
    frozen = ('moving_mean', 'moving_variance')
    P = {k: torch.tensor(v, dtype=torch.float32, requires_grad=not k.endswith(frozen)) for k, v in p.items()}
    moving = {k: v.detach().clone() for k, v in P.items() if k.endswith(frozen)}
    passes = [cases.images(2, 32, 48, 30 + i, 40 + i)[0] for i in range(npasses)]
    got = _graph_moving_after(passes, P, moving)
    want = {k: np.asarray(v, dtype=np.float64) for k, v in p.items() if k.endswith(frozen)}
    biased = dict(want)
    for im in passes:
        rec = {}
        x = torch.from_numpy(2 * (im.astype(np.float64) / 255.0) - 1.0).permute(0, 3, 1, 2)
        rt.encoder(rt.Ops(p, torch.float64, bn_record=rec), x, 'cnet', 'batch', True)
        want.update(train_ref.bn_moving_update(want, rec))
        biased.update(train_ref.bn_moving_update(biased, {k: (m, v, 1 << 60) for k, (m, v, _) in rec.items()}))
    worst, resolved = 0.0, []
    for k in sorted(k for k in want if k.startswith('cnet.')):
        g, w, b = got[k].double().numpy(), want[k], biased[k]
        err = float(np.abs(g - w).max())
        tol = 2e-7 * (npasses + 1) * float(np.abs(w).max())     # fp32 statistics: ~1e-7 relative per pass
        assert err <= tol, f'{k}: {err:.3e} > {tol:.3e}'
        worst = max(worst, err / float(np.abs(w).max()))
        gap = float(np.abs(b - w).max())                          # what the biased rule would be off by
        if k.endswith('moving_variance') and gap > 4 * tol:
            assert float(np.abs(g - b).max()) >= 0.5 * gap, f'{k} follows the biased-variance rule'
            resolved.append(k)
    print(f'{npasses} pass(es): worst relative error {worst:.2e}; the biased rule is told apart on {len(resolved)} of '
          f'15 layers')
    # every layer after the stem: at n = 768 the stem's variance is too small for its 1/767 to clear fp32 rounding
    assert len(resolved) >= 14


def test_torch_backend_encoder_moving_statistics_follow_keras():
    """The torch-backend BasicEncoder (batch norm) in training mode follows the same rule over three calls."""
    from tf_raft_b200.layers.extractor import BasicEncoder
    p = weights.init_params('raft', 21, bias_scale=0.05, norm_jitter=0.1)
    enc = BasicEncoder(output_dim=256, norm_type='batch', device='cpu', backend='torch')
    enc.load_params({k: v.copy() for k, v in p.items()}, 'cnet.')      # the layer updates its moving statistics in place
    want = {k: np.asarray(v, dtype=np.float64) for k, v in p.items() if k.endswith(('moving_mean', 'moving_variance'))}
    for i in range(3):
        im = cases.images(2, 32, 48, 30 + i, 40 + i)[0]
        enc(torch.from_numpy(im), training=True, raw_image=True)
        rec = {}
        x = torch.from_numpy(2 * (im.astype(np.float64) / 255.0) - 1.0).permute(0, 3, 1, 2)
        rt.encoder(rt.Ops(p, torch.float64, bn_record=rec), x, 'cnet', 'batch', True)
        want.update(train_ref.bn_moving_update(want, rec))
    got = enc.state_dict('cnet.')
    for k in (k for k in want if k.startswith('cnet.')):
        w = want[k]
        assert float(np.abs(got[k].double().numpy() - w).max()) <= 8e-7 * float(np.abs(w).max()), k
