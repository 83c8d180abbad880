"""The training step's state over several steps, against the float64 restatement of oracle/train_ref.py.

`test_train.py` checks one step (t = 1), where Adam's update is lr * g / (|g| + eps'): almost independent of the
gradient's scale, of the clip, of the bias correction and of what m and v hold.  The tests below run the kernels and the
host glue of the training step for several steps, with clipping that switches on and off, weight decay large enough to
see and a learning rate that changes every step:

a. `raft_b200_sumsq` against the fp64 sum, within the fp32 bound of the kernel's own summation order, bit-reproducible;
b. `raft_b200_adamw_step` over 6 steps against the restatement running free from the same fp32 start: p, m and v;
c. `FlatState.apply` (schedule index, bias correction, slice padding) over 8 steps;
d. `_CorrPyramid.backward` against torch.autograd of the oracle correlation in float64;
e. three `RAFT.train_step`s against three oracle steps (CPU autograd + the restatement, carrying m, v, t and the
   BatchNorm moving statistics);
f. the trained values reaching inference, with and without CUDA graphs.

Each comparison prints the worst error; where an fp32 NumPy restatement exists, also its error against the same fp64
truth, which shows how much of the tolerance fp32 arithmetic needs by itself.
"""
import math

import numpy as np
import pytest
import torch

import cases
from oracle import raft_torch as rt, train_ref, weights

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, torch.float64
U = 2.0 ** -24                                   # fp32 unit roundoff
B1, B2, EPS = 0.9, 0.999, 1e-7
# what the AdamW kernel receives: 1 - fp32(0.999) is 1.3e-5 below 1e-3 (as in TensorFlow, whose beta_2 is an fp32 variable)
B1_32, B2_32, EPS_32 = (float(np.float32(x)) for x in (B1, B2, EPS))
FROZEN = ('moving_mean', 'moving_variance')


@pytest.fixture(scope='module')
def L():
    from tf_raft_b200 import _lib
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    return _lib


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).cuda()


def host(t):
    return t.detach().cpu().double().numpy()


# --------------------------------------------------------------------------------------------- a. global sum of squares
SUMSQ_SIZES = (0, 1, 7, 255, 256, 257, 135167, 135168, 135169, 540673, 5260420)
PARTIAL_CAP = 132 * 4                            # partial blocks: 4 per SM of an H100 (raft_b200_sumsq)


def _mixed(n, seed):
    """normal x 10^U(-6, 2), one entry in ten exactly 0."""
    rng = np.random.default_rng(seed)
    g = rng.standard_normal(n) * 10.0 ** rng.uniform(-6, 2, n)
    g[rng.uniform(size=n) < 0.1] = 0.0
    return g.astype(F32)


def _sumsq(L, g, n, npartials):
    part = torch.full((npartials,), float('nan'), device='cuda')       # only the partials the kernel writes may be read
    out = torch.full((1,), float('nan'), device='cuda')
    L.check(L.lib().raft_b200_sumsq(L.ptr(g), n, L.ptr(part), npartials, L.ptr(out), L.stream()), 'sumsq')
    return out


def _sumsq_chain(n, npartials):
    """Longest chain of fp32 roundings in raft_b200_sumsq's order: each thread's strided serial sum (with its squares),
    the 5-level warp tree, the 8 warp sums in series -- once over the elements, once over the partials."""
    blocks = max(1, min(npartials, PARTIAL_CAP, -(-n // 256)))
    return (-(-n // (blocks * 256)) + 1) + 5 + 8 + -(-blocks // 256) + 5 + 8


@pytest.fixture(scope='module')
def mixed_data():
    cache = {}

    def get(n):
        if n not in cache:
            g = _mixed(n, 100 + n)
            cache[n] = (g, float(np.square(g.astype(np.float64)).sum()))
        return cache[n]
    return get


@pytest.mark.parametrize('npartials', (1, 3, 528, 1024))
@pytest.mark.parametrize('n', SUMSQ_SIZES)
def test_sumsq_vs_fp64(L, mixed_data, n, npartials):
    """sum g^2 over sizes around the block (256) and grid (528 x 256) boundaries up to RAFT's flat buffer, within the
    summation bound chain * 2^-24 * sum, and bit-identical over repeated calls."""
    g, truth = mixed_data(n)
    buf = dev(g) if n else torch.full((1,), float('nan'), device='cuda')     # n = 0 must not read the buffer
    got = [float(_sumsq(L, buf, n, npartials)) for _ in range(3)]
    assert got[0] == got[1] == got[2], f'not deterministic: {got}'
    if n == 0:
        assert got[0] == 0.0
        return
    bound = 1.01 * _sumsq_chain(n, npartials) * U * truth
    err = abs(got[0] - truth)
    np32 = abs(float(np.square(g).sum(dtype=F32)) - truth)
    print(f'sumsq n={n} npartials={npartials}: rel error {err / truth:.2e} (fp32 NumPy {np32 / truth:.2e}), '
          f'bound {bound / truth:.2e}')
    assert err <= bound, (err, bound)


# --------------------------------------------------------------------------------------------- b. AdamW kernel, 6 steps
FACTORS = (10.0, 0.5, 3.0, 0.01, 2.0, 0.2, 5.0, 0.8)        # global norm of each step's gradient, in units of CLIP
CLIP = 1.0
LRS = (1e-3, 2e-3, 5e-4, 1e-3, 3e-3, 1e-3)


def _grad_sequence(n, steps, seed):
    """fp32 gradients whose global norm is FACTORS[k] * CLIP at step k; 30 % of the entries flip sign from step to
    step, one in eleven is 0 at every step (its v stays 0), one in thirteen is ~1e-7 (near epsilon)."""
    rng = np.random.default_rng(seed)
    base = rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 0, n)
    zero = np.arange(n) % 11 == 5
    tiny = np.arange(n) % 13 == 6
    out = []
    for k in range(steps):
        base = np.where(rng.uniform(size=n) < (0.3 if k else 0.0), -base, base)
        g = base * FACTORS[k] * CLIP / np.sqrt(np.square(base).sum())
        g[zero] = 0.0
        g[tiny] = np.sign(base[tiny]) * 1e-7 * rng.uniform(0.5, 2.0, int(tiny.sum()))
        out.append(g.astype(F32))
    return out


def _adam_fp32(p, m, v, g, sumsq, clip, lr_t, wd):
    """adamw_kernel's arithmetic restated in fp32 NumPy (for the printed comparison only)."""
    f = F32
    scale = f(1)
    if clip > 0:
        norm = np.sqrt(f(sumsq))
        scale = f(clip) / max(norm, f(clip))
    gi = g * scale
    w = p - f(wd) * p
    b1, b2 = f(B1), f(B2)
    m = b1 * m + (f(1) - b1) * gi
    v = b2 * v + (f(1) - b2) * gi * gi
    return w - f(lr_t) * m / (np.sqrt(v) + f(EPS)), m, v


@pytest.mark.parametrize('wd', (0.0, 1e-2))
@pytest.mark.parametrize('clip', ('active', 'inactive', 'disabled'))
@pytest.mark.parametrize('n', (1, 1023, 540673))
def test_adamw_kernel_six_steps_vs_fp64(L, n, clip, wd):
    """Six clipped AdamW steps on one flat buffer (n = 540673 is above the kernel's grid-stride cap of 2112 x 256).  The
    gradient norm changes every step, so an active clip scales some steps and not others; p, m and v are compared with
    the restatement after every step, which is given the kernel's own fp32 hyperparameters (beta, epsilon, wd, lr_t).
    Tolerance per entry at step t: for p, 4 t + 8 roundings of |p| + 4 sum(lr_t) (the
    largest the Adam terms can have moved it); for m and v, 4 t + 2 chain roundings of their magnitude, chain = the sum
    of squares' rounding chain, whose error the clip scale inherits (m / sqrt(v) does not, up to epsilon)."""
    clip_norm = {'active': CLIP, 'inactive': 1e3 * CLIP, 'disabled': 0.0}[clip]
    rng = np.random.default_rng(n)
    p0 = (rng.standard_normal(n) * 0.1).astype(F32)
    p0[::7] = 0.0
    grads = _grad_sequence(n, len(LRS), seed=n + 1)
    P, G, M, V = dev(p0), torch.empty(n, device='cuda'), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
    ref = train_ref.AdamW(float(np.float32(wd)), 0.0, B1_32, B2_32, EPS_32)
    want = {'x': p0.astype(np.float64)}
    p32, m32, v32 = p0.copy(), np.zeros(n, F32), np.zeros(n, F32)
    mag_m = np.zeros(n)
    upd = 0.0
    chain = _sumsq_chain(n, 1024)
    worst, worst32 = dict(p=0.0, m=0.0, v=0.0), dict(p=0.0, m=0.0, v=0.0)
    for k, (g, lr) in enumerate(zip(grads, LRS)):
        t = k + 1
        ref.learning_rate = lr
        lr_t = float(np.float32(ref.lr_t()))
        ref.learning_rate *= lr_t / ref.lr_t()              # the restatement steps with the fp32 lr_t the kernel gets
        G.copy_(torch.from_numpy(g))
        sumsq = _sumsq(L, G, n, 1024)
        L.check(L.lib().raft_b200_adamw_step(L.ptr(P), L.ptr(G), L.ptr(M), L.ptr(V), n, L.ptr(sumsq), float(clip_norm),
                                             float(lr_t), B1, B2, EPS, float(wd), L.stream()), 'adamw_step')
        p32, m32, v32 = _adam_fp32(p32, m32, v32, g, float(sumsq), clip_norm, lr_t, wd)
        want = ref.apply(want, {'x': g}, clip_norm)
        scale = train_ref.clip_scale(train_ref.global_sumsq([g]), clip_norm)
        mag_m = B1 * mag_m + (1 - B1) * np.abs(g.astype(np.float64)) * scale
        upd += lr_t * 4.0                                   # |m / (sqrt(v) + eps)| < 3.2 for these betas
        c = (4 * t + 2 * chain) * U                         # m, v: scaled by the clip, which inherits sumsq's error
        tol = dict(p=(4 * t + 8) * U * (np.abs(want['x']) + upd), m=c * mag_m + 1e-45, v=c * ref.v['x'] + 1e-45)
        truth = dict(p=want['x'], m=ref.m['x'], v=ref.v['x'])
        for key, got, got32 in (('p', P, p32), ('m', M, m32), ('v', V, v32)):
            e = np.abs(host(got) - truth[key])
            e32 = np.abs(got32.astype(np.float64) - truth[key])
            worst[key] = max(worst[key], float((e / tol[key]).max()))
            worst32[key] = max(worst32[key], float((e32 / tol[key]).max()))
            bad = np.flatnonzero(e > tol[key])
            assert bad.size == 0, (f'step {t}: {key}[{bad[0]}] = {host(got)[bad[0]]!r}, want {truth[key][bad[0]]!r} '
                                   f'(tolerance {tol[key][bad[0]]:.3e}, {bad.size} entries out)')
    print(f'adamw n={n} clip={clip} wd={wd}: worst error / tolerance ' +
          ', '.join(f'{k} {worst[k]:.3f} (fp32 NumPy {worst32[k]:.3f})' for k in worst))


# --------------------------------------------------------------------------------------------- c. FlatState.apply
GLUE_SHAPES = {'a': (1,), 'b': (3,), 'c': (1, 5), 'd': (17,), 'e': (4099,)}


@pytest.mark.parametrize('schedule', ('cyclical', 'constant'))
def test_flat_state_apply_eight_steps(L, schedule):
    """FlatState + AdamW on odd-sized variables (16-byte padding between the slices) for 8 steps: with the cyclical
    schedule (step size 3, through the end of its first cycle) and a clip, then with a constant lr and no clip.  Every
    variable follows the restatement, which evaluates the schedule at iterations - 1 = t - 1 and corrects the bias with
    t; the padding of p, m and v stays 0.  The restatement keeps the host's hyperparameters (beta_2 = 0.999): the kernel's
    fp32 beta_2 moves v by up to 1.3e-5 relative and the Adam term by half that, so the tolerances of the kernel test
    gain 2e-5 of v and 1e-5 of the Adam terms."""
    from tf_raft_b200.train import AdamW, CyclicalLearningRate, FlatState, first_cycle_scaler
    rng = np.random.default_rng(77)
    init = {k: (rng.standard_normal(s) * 0.1).astype(F32) for k, s in GLUE_SHAPES.items()}
    flat = FlatState({k: dev(v) for k, v in init.items()}, lambda k: True)
    if schedule == 'cyclical':
        lr, clip_norm = CyclicalLearningRate(1e-3, 2e-3, step_size=3, scale_fn=first_cycle_scaler), CLIP
        ref = train_ref.AdamW(1e-2, lambda s: train_ref.cyclical_lr(s, 1e-3, 2e-3, 3, first_cycle_scaler))
    else:
        lr, clip_norm = 2e-3, None
        ref = train_ref.AdamW(1e-2, 2e-3)
    opt = AdamW(weight_decay=1e-2, learning_rate=lr)
    n = sum(int(np.prod(s)) for s in GLUE_SHAPES.values())
    seq = _grad_sequence(n, 8, seed=5)
    pad = torch.ones(flat.p.numel(), dtype=torch.bool)
    for o, k in zip(flat.offsets, flat.names):
        pad[o:o + init[k].size] = False
    assert int(pad.sum()) == 3 + 1 + 3 + 3 + 1                        # 1->4, 3->4, 5->8, 17->20, 4099->4100
    want = {k: v.astype(np.float64) for k, v in init.items()}
    upd, worst = 0.0, 0.0
    for s in range(8):
        flat.zero_grad()
        grads, pos = {}, 0
        for k, shp in GLUE_SHAPES.items():
            sz = int(np.prod(shp))
            grads[k] = seq[s][pos:pos + sz].reshape(shp)
            flat.views[k].grad.copy_(torch.from_numpy(grads[k]))
            pos += sz
        flat.apply(opt, clip_norm)
        upd += ref.lr_t() * 4.0
        want = ref.apply(want, grads, clip_norm)
        assert opt.iterations == ref.iterations == s + 1
        c_p, c = (4 * (s + 1) + 8) * U, (4 * (s + 1) + 2 * _sumsq_chain(n, 1024)) * U     # as in the kernel test
        for k in GLUE_SHAPES:
            o = flat.offsets[flat.names.index(k)]
            sz = init[k].size
            # m crosses 0 where the gradient flips sign: its rounding is relative to the tensor's scale, not the entry's
            for name, got, truth, tol in (('p', flat.p, want[k], c_p * (np.abs(want[k]) + upd) + 1e-5 * upd),
                                          ('m', flat.m, ref.m[k], c * (np.abs(ref.m[k]) + np.abs(ref.m[k]).max())),
                                          ('v', flat.v, ref.v[k], (c + 2e-5) * ref.v[k] + 1e-45)):
                g = host(got[o:o + sz]).reshape(truth.shape)
                err = np.abs(g - truth)
                worst = max(worst, float((err / tol).max()))
                assert (err <= tol).all(), f'step {s + 1} {name} of {k}: max error {err.max():.3e}'
        for buf in (flat.p, flat.m, flat.v):
            assert not bool(buf.cpu()[pad].any()), 'padding entries changed'
    print(f'FlatState.apply ({schedule}): worst error / tolerance {worst:.3f}')


# --------------------------------------------------------------------------------------------- d. correlation backward
BWD_CASES = tuple(c for c in cases.PYRAMID_CASES if c in ((3, 9, 13, 64, 1), (3, 19, 23, 256, 4), (2, 31, 31, 256, 5)))


@pytest.mark.parametrize('precision', ('f16x2', 'fp32'))
@pytest.mark.parametrize('case', BWD_CASES, ids=lambda c: 'x'.join(map(str, c)))
def test_corr_pyramid_backward_vs_fp64(L, case, precision):
    """d fmap1, d fmap2 of the correlation pyramid (fp32 GEMMs on the pooled features) against torch.autograd of the
    oracle CorrBlock in float64, with a random upstream gradient on every level; 1, 4 and 5 levels, odd sizes, C = 64 and
    256.  Tolerance: the pyramid's 2e-5 abs + 2e-5 rel, the abs part scaled to the gradient's largest entry."""
    from tf_raft_b200.train import _CorrPyramid
    b, h, w, c, levels = case
    f1, f2 = cases.fmaps(b, h, w, c, seed=30 + c + levels)
    rng = np.random.default_rng(levels)
    ups = [rng.standard_normal((b * h * w, lh, lw, 1)).astype(F32) for lh, lw in cases.level_sizes(h, w, levels)]
    g1, g2 = dev(f1).requires_grad_(True), dev(f2).requires_grad_(True)
    pyr = _CorrPyramid.apply(g1, g2, levels, 4, precision)
    got = torch.autograd.grad(pyr, (g1, g2), [dev(u) for u in ups])
    res = {}
    for dtype in (F64, torch.float32):
        t1 = torch.from_numpy(f1).to(dtype).requires_grad_(True)
        t2 = torch.from_numpy(f2).to(dtype).requires_grad_(True)
        res[dtype] = torch.autograd.grad(rt.CorrBlock(t1, t2, levels, 4).corr_pyramid, (t1, t2),
                                         [torch.from_numpy(u).to(dtype) for u in ups])
    for i, name in enumerate(('fmap1', 'fmap2')):
        truth = res[F64][i].numpy()
        scale = float(np.abs(truth).max())
        err = np.abs(host(got[i]) - truth)
        err32 = float(np.abs(res[torch.float32][i].double().numpy() - truth).max())
        print(f'corr backward {precision} {case} d{name}: max-abs {err.max():.2e} (fp32 oracle {err32:.2e}), '
              f'scale {scale:.2f}')
        tol = 2e-5 * scale + 2e-5 * np.abs(truth)
        assert (err <= tol).all(), f'd{name}: max error {err.max():.3e} at scale {scale:.3e}'


# --------------------------------------------------------------------------------------------- e. three training steps
def _oracle_grads(params, im1, im2, flow_gt, valid, variant, iters):
    """Loss, gradient of every trainable variable and BatchNorm batch statistics of one oracle forward (CPU fp32,
    torch.autograd), the sequence loss written out (losses.py:4-24)."""
    leaves = {k: torch.tensor(np.asarray(v), dtype=torch.float32, requires_grad=not k.endswith(FROZEN))
              for k, v in params.items()}
    rec = {}
    preds = rt.forward(leaves, im1, im2, variant, iters, training=True, bn_record=rec)
    fg, va = torch.from_numpy(flow_gt), torch.from_numpy(valid)
    vm = (va & (torch.sqrt((fg ** 2).sum(-1)) < 400)).float().unsqueeze(-1)
    loss = sum(0.8 ** (iters - i - 1) * (vm * (p - fg).abs()).mean() for i, p in enumerate(preds))
    names = [k for k, v in leaves.items() if v.requires_grad]
    grads = torch.autograd.grad(loss, [leaves[k] for k in names])
    return float(loss), {k: g.double().numpy() for k, g in zip(names, grads)}, rec


TRAIN_CLIP = {'small': 25.0, 'raft': 20.0}       # below the global gradient norm of each of the three steps (printed)


@pytest.mark.parametrize('variant,iters', [('small', 3), ('raft', 2)])
def test_three_train_steps_vs_oracle(L, variant, iters):
    """Three RAFT.train_steps at 64x96, batch 2, with a clip below the gradient norm, wd = 1e-3 and a cyclical lr that
    changes every step, against three oracle steps: per step the loss, the global norm, the update where the gradient is
    well determined, and (RAFT) the moving statistics of every cnet BatchNorm layer.

    Each oracle gradient is taken at the model's parameters before the step: Adam's update of an entry whose gradient is
    decided by rounding is +-lr either way, so two free-running trajectories would part by that much.  m, v, t, the
    schedule and the moving statistics are the restatement's own, carried from step to step."""
    import tf_raft_b200 as T
    from tf_raft_b200.train import AdamW, CyclicalLearningRate, first_cycle_scaler
    bsz, H, W = 2, 64, 96
    p = weights.init_params(variant, 21, bias_scale=0.05, norm_jitter=0.1)
    model = (T.RAFT if variant == 'raft' else T.SmallRAFT)(iters=iters, iters_pred=iters, precision='f16x2')
    model.load_params(p)
    wd, clip_norm = 1e-3, TRAIN_CLIP[variant]
    model.compile(optimizer=AdamW(weight_decay=wd, learning_rate=CyclicalLearningRate(1e-4, 3e-4, step_size=2)),
                  clip_norm=clip_norm)
    ref = train_ref.AdamW(wd, lambda s: train_ref.cyclical_lr(s, 1e-4, 3e-4, 2, first_cycle_scaler))
    cur = {k: np.asarray(v, dtype=F32) for k, v in p.items()}
    moving_ref = {k: v.astype(np.float64) for k, v in cur.items() if k.endswith(FROZEN)}
    rng = np.random.default_rng(9)
    worst_upd = worst_mov = 0.0
    for step in range(3):
        im1, im2 = cases.images(bsz, H, W, 3 + 2 * step, 4 + 2 * step)
        flow_gt = (rng.standard_normal((bsz, H, W, 2)) * 5).astype(F32)
        valid = rng.uniform(size=(bsz, H, W)) > 0.1
        loss_o, grads_o, rec = _oracle_grads(cur, im1, im2, flow_gt, valid, variant, iters)
        norm_o = math.sqrt(train_ref.global_sumsq(grads_o))
        lr = ref.lr()
        want = ref.apply({k: cur[k] for k in grads_o}, grads_o, clip_norm)
        moving_ref.update(train_ref.bn_moving_update(moving_ref, rec))
        model.reset_metrics()
        out = model.train_step((dev(im1), dev(im2), dev(flow_gt), torch.from_numpy(valid).cuda()))
        tr = model._trainer
        assert model.optimizer.iterations == step + 1
        assert out['loss'] == pytest.approx(loss_o, rel=2e-4), (step, out['loss'], loss_o)
        gnorm = math.sqrt(float((tr.flat.g.double() ** 2).sum()))
        assert gnorm == pytest.approx(norm_o, rel=1e-3), (step, gnorm, norm_o)
        assert norm_o > clip_norm, 'the clip must be active'
        new = {k: host(v) for k, v in tr.flat.views.items()}
        for k, w in want.items():
            g = np.abs(grads_o[k])
            sel = g >= 0.2 * g.max()
            if float(g.max()) < 1e-5:                                # zero true gradient: noise
                continue
            err = float(np.abs((new[k] - cur[k]) - (w - cur[k]))[sel].max()) / lr
            worst_upd = max(worst_upd, err)
            assert err <= 5e-2, f'step {step + 1} {k}: update differs by {err:.3f} x lr'
        decay = max(float(np.abs(wd * cur[k]).max()) for k in want) / lr
        if variant == 'raft':
            for k, w in moving_ref.items():
                got = host(tr.moving[k])
                err = float(np.abs(got - w).max()) / float(np.abs(w).max())
                worst_mov = max(worst_mov, err)
                assert err <= 2e-6, f'step {step + 1} {k}: relative error {err:.2e}'
        print(f'{variant} step {step + 1}: loss {out["loss"]:.6f} (oracle {loss_o:.6f}), norm {gnorm:.3f} '
              f'(oracle {norm_o:.3f}, clip {clip_norm}), lr {lr:.2e}, largest decay {decay:.2f} x lr')
        cur = {k: (new[k].astype(F32) if k in new else host(tr.moving[k]).astype(F32)) for k in cur}
    print(f'{variant}: worst update error {worst_upd:.3f} x lr, worst moving-statistics error {worst_mov:.2e} relative')


# --------------------------------------------------------------------------------------------- f. hand-off to inference
@pytest.mark.parametrize('use_graph', (False, True), ids=('eager', 'graph'))
@pytest.mark.parametrize('variant', ('small', 'raft'))
def test_trained_weights_reach_inference(L, variant, use_graph):
    """After two train_steps the next inference call runs on the trained values: its output equals a fresh model loaded
    with the trained state_dict, and differs from the output before training (a CUDA graph captured before training
    must not be replayed).  An inference call between steps leaves the training state untouched, and the following step
    runs as step 3 on the carried moments."""
    import tf_raft_b200 as T
    from tf_raft_b200.train import AdamW
    cls = T.RAFT if variant == 'raft' else T.SmallRAFT
    iters = 2
    p = weights.init_params(variant, 21, bias_scale=0.05, norm_jitter=0.1)
    model = cls(iters=iters, iters_pred=iters, precision='f16x2', use_graph=use_graph)
    model.load_params(p)
    model.compile(optimizer=AdamW(weight_decay=1e-3, learning_rate=1e-3), clip_norm=1.0)
    im1, im2 = (dev(a) for a in cases.images(2, 64, 96, 3, 4))
    rng = np.random.default_rng(9)
    data = (im1, im2, dev((rng.standard_normal((2, 64, 96, 2)) * 5).astype(F32)),
            torch.from_numpy(rng.uniform(size=(2, 64, 96)) > 0.1).cuda())
    before = model([im1, im2], training=False, last_only=True)[-1].clone()    # captures the graph when use_graph
    model.train_step(data)
    model.train_step(data)
    tr = model._trainer
    snap = dict(m=tr.flat.m.clone(), v=tr.flat.v.clone(), p=tr.flat.p.clone(),
                moving={k: v.clone() for k, v in tr.moving.items()})
    got = model([im1, im2], training=False, last_only=True)[-1].clone()
    assert model._trainer is tr and model.optimizer.iterations == 2
    assert torch.equal(tr.flat.m, snap['m']) and torch.equal(tr.flat.v, snap['v']) and torch.equal(tr.flat.p, snap['p'])
    assert all(torch.equal(tr.moving[k], v) for k, v in snap['moving'].items())
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    trained = tr.params()
    assert sorted(sd) == sorted(trained)
    for k, v in trained.items():
        assert torch.equal(sd[k], v), f'{k}: state_dict is not the trained value'
    fresh = cls(iters=iters, iters_pred=iters, precision='f16x2', use_graph=use_graph)
    fresh.load_params(sd)
    want = fresh([im1, im2], training=False, last_only=True)[-1]
    assert torch.equal(got, want)
    assert not torch.equal(got, before)
    # step 3 continues from the carried state: m = b1 m_2 + (1 - b1) * clipped g_3
    model.train_step(data)
    assert model._trainer is tr and model.optimizer.iterations == 3
    g3 = tr.flat.g
    scale = min(1.0, 1.0 / math.sqrt(float((g3.double() ** 2).sum())))
    m3 = B1 * snap['m'].double() + (1 - B1) * scale * g3.double()
    err = float((tr.flat.m.double() - m3).abs().max())
    print(f'{variant} use_graph={use_graph}: step 3 m error {err:.2e} (|m| up to {float(m3.abs().max()):.2e})')
    assert err <= 1e-5 * float(m3.abs().max())
