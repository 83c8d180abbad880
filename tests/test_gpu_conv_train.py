"""The training step's tensor-core convolutions (raft_b200_conv_tc_forward / _backward, train_precision='f16x2') against
fp64, at every eligible layer shape of both variants (conv_train_cases), and the f16x2 training step under the unchanged
gates of the existing one-step and three-step oracle tests (and, self-supervised, against the fp32 step).

E is the fp64 value of the three-pass product on the split operands (hi.hi' + hi.lo' + lo.hi', scaled back), the model
of test_gpu_mainloop.py.  On small integers every product is a multiple of the scales and E is exact: outputs equal it
bit for bit.  On N(0, 1) data and on gradient-like N(0, 1) * 1e-6 data, |got - E| <= 2u (L + n_groups + 2 + slices) S,
u = 2^-24, S = sum |products|, L the MMA chain of a promotion group (forward and input gradient: 12 * 2; weight
gradient: 24 per 128-pixel tile * 2) and `slices` the weight gradient's ordered slice sum (0 otherwise)."""
import ctypes
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_train_cases

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
WORST = {}


def _lib():
    from tf_raft_b200 import _lib, build
    build.build()
    return _lib


def run(x, k, b, g, need_dx=True):
    """(out, grad_x, grad_kernel) of the library on NHWC x, HWIO k, bias b, NHWC grad_out g (fp32 CUDA tensors)."""
    L = _lib()
    B, H, W, cin = x.shape
    kh, kw, _, cout = k.shape
    dims = (B, H, W, cin, kh, kw, cout)
    need = ctypes.c_size_t()
    L.call('conv_tc_forward', x.device, None, None, None, *dims, None, None, None, ctypes.byref(need))
    ws = L.workspace(need.value, x.device)
    nb = ctypes.byref(ctypes.c_size_t(ws.numel()))
    planes = torch.empty(2 * B * H * W * ((cin + 63) // 64 * 64) + 128, dtype=torch.float16, device=x.device)
    out = torch.empty((B, H, W, cout), device=x.device)
    L.call('conv_tc_forward', x.device, L.ptr(x), L.ptr(k), L.ptr(b), *dims, L.ptr(out), L.ptr(planes), L.ptr(ws), nb)
    dx = torch.empty_like(x) if need_dx else None
    dk = torch.empty_like(k)
    L.call('conv_tc_backward', x.device, L.ptr(planes), L.ptr(k), L.ptr(g), *dims, L.ptr(dx), L.ptr(dk), L.ptr(ws), nb)
    return out, dx, dk


def _k(t):
    m = float(t[torch.isfinite(t)].abs().max()) if torch.isfinite(t).any() else 0.0
    return 0 if m == 0 else 13 - math.frexp(m)[1]


def _split(t, k):
    s = (t * 2.0 ** k).to(torch.float32)
    hi = s.half()
    lo = (s - hi.float()).half()
    return hi.double(), lo.double()


def expected(x, k, b, g, kw_clamp=24, kg_clamp=100):
    """fp64 (E, S) of forward, input gradient and weight gradient; tensors NCHW / OIHW inside."""
    kh, kwd = k.shape[0], k.shape[1]
    pad = ((kh - 1) // 2, (kwd - 1) // 2)
    xs = x.permute(0, 3, 1, 2)
    ws = k.permute(3, 2, 0, 1)
    gs = g.permute(0, 3, 1, 2)
    k_w = max(-kw_clamp, min(kw_clamp, _k(k)))
    k_g = max(-kg_clamp, min(kg_clamp, _k(g)))
    k_x = max(-kg_clamp, min(kg_clamp, _k(x)))
    xh, xl = _split(xs, k_x)
    wh, wl = _split(ws, k_w)
    gh, gl = _split(gs, k_g)
    conv = lambda a, w: F.conv2d(a, w, padding=pad)
    dinp = lambda gg, w: torch.nn.grad.conv2d_input(xs.shape, w, gg, padding=pad)
    dwt = lambda a, gg: torch.nn.grad.conv2d_weight(a, ws.shape, gg, padding=pad)
    fwd = (conv(xh, wh) + conv(xh, wl) + conv(xl, wh)) * 2.0 ** -(k_w + k_x) + b.double().view(1, -1, 1, 1)
    dx = (dinp(gh, wh) + dinp(gh, wl) + dinp(gl, wh)) * 2.0 ** -(k_w + k_g)
    dw = (dwt(xh, gh) + dwt(xl, gh) + dwt(xh, gl)) * 2.0 ** -(k_g + k_x)
    ax, aw, ag = xs.double().abs(), ws.double().abs(), gs.double().abs()
    S = (conv(ax, aw) + b.double().abs().view(1, -1, 1, 1), dinp(ag, aw), dwt(ax, ag))
    nhwc = lambda t: t.permute(0, 2, 3, 1)
    hwio = lambda t: t.permute(2, 3, 1, 0)
    return (nhwc(fwd), nhwc(dx), hwio(dw)), (nhwc(S[0]), nhwc(S[1]), hwio(S[2]))


def plan(B, H, W, cin, kh, kw, cout):
    """(n_groups forward, n_groups input gradient, n_groups weight gradient, slices) as conv_train.cuh plans them."""
    def tile(h, w):
        best = None
        for t in (128, 64, 32, 16, 8):
            area = -(-w // t) * t * (-(-h // (128 // t)) * (128 // t))
            if best is None or area < best[0]:
                best = (area, t, 128 // t)
        return best[1], best[2]
    tw, th = tile(H, W)
    ptiles = B * -(-W // tw) * -(-H // th)
    cin_pad, cout_pad = -(-cin // 64) * 64, -(-cout // 64) * 64
    base = kh * kw * -(-cout_pad // 128) * (cin_pad // 64)
    slices = min(max(-(-256 // base), 1), ptiles)
    tps = -(-ptiles // slices)
    slices = -(-ptiles // tps)
    return -(-kh * kw * cin_pad // 64 // 2), -(-kh * kw * cout_pad // 64 // 2), -(-tps // 2), slices


def check(case, kind, got, E, S, groups, slices):
    names = ('forward', 'grad_x', 'grad_kernel')
    for i, (a, e, s) in enumerate(zip(got, E, S)):
        a = a.double()
        if kind == 'integer':
            assert torch.equal(a, e), f'{case} {names[i]}: {int((a != e).sum())} outputs differ from the exact sum'
            continue
        L = 24 if i < 2 else 48
        bound = 2 * U * (L + groups[i] + 2 + (slices if i == 2 else 0)) * s
        err = (a - e).abs()
        ratio = float((err / bound.clamp_min(1e-300)).max())
        WORST[(kind, names[i])] = max(WORST.get((kind, names[i]), (0.0, ''))[0], ratio), case
        assert ratio <= 1.0, f'{case} {names[i]}: worst |got - E| / bound = {ratio:.3f}'


def data(kind, B, H, W, cin, kh, kw, cout, seed):
    gen = torch.Generator(device='cuda').manual_seed(seed)
    if kind == 'integer':
        r = lambda *s: torch.randint(-2, 3, s, generator=gen, device='cuda').float()
        return r(B, H, W, cin), r(kh, kw, cin, cout), r(cout), r(B, H, W, cout)
    n = lambda *s: torch.randn(*s, generator=gen, device='cuda')
    gscale = 1e-6 if kind == 'gradlike' else 1.0
    return n(B, H, W, cin), n(kh, kw, cin, cout) * 0.1, n(cout) * 0.1, n(B, H, W, cout) * gscale


CASES = conv_train_cases.cases()


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_against_fp64(case):
    name, B, H, W, cin, kh, kw, cout = case
    ng_f, ng_d, ng_w, slices = plan(B, H, W, cin, kh, kw, cout)
    for i, kind in enumerate(('integer', 'normal', 'gradlike')):
        x, k, b, g = data(kind, B, H, W, cin, kh, kw, cout, seed=zlib.crc32(name.encode()) % 1000 + i)
        got = run(x, k, b, g)
        E, S = expected(x, k, b, g)
        check(name, kind, got, E, S, (ng_f, ng_d, ng_w), slices)
        del got, E, S
    torch.cuda.empty_cache()


def test_worst_ratios_printed():
    for (kind, what), (r, case) in sorted(WORST.items()):
        print(f'conv_train {kind} {what}: worst |got - E| / bound {r:.4f} ({case})')


@pytest.mark.parametrize('case', [c for c in CASES if c[0].startswith('ragged')][:6], ids=lambda c: c[0])
def test_nan_reaches_exactly_its_outputs_and_calls_repeat_bit_for_bit(case):
    name, B, H, W, cin, kh, kw, cout = case
    x, k, b, g = data('normal', B, H, W, cin, kh, kw, cout, seed=5)
    ref = run(x, k, b, g)
    again = run(x, k, b, g)
    for a, r in zip(again, ref):
        assert torch.equal(a, r), f'{name}: two calls differ'
    # at the bottom-right corner, where a ragged tile overhangs the image: the kernel zeroes the x rows that meet the
    # gradient's zero-filled rows there, so the x entry reaches no weight-gradient tap whose sum does not include it
    px = (B - 1, H - 1, W - 1, cin // 3)
    pg = (0, H - 1, W - 1, cout // 2)
    xn, gn = x.clone(), g.clone()
    xn[px] = float('nan')
    gn[pg] = float('nan')
    out, dx, dk = run(xn, k, b, gn)
    # which outputs include the planted entries: the same sums on 0/1 indicators in fp64
    ix = torch.zeros_like(x, dtype=torch.float64); ix[px] = 1
    ig = torch.zeros_like(g, dtype=torch.float64); ig[pg] = 1
    pad = ((kh - 1) // 2, (kw - 1) // 2)
    ones_w = torch.ones((cout, cin, kh, kw), dtype=torch.float64, device='cuda')
    reach_out = F.conv2d(ix.permute(0, 3, 1, 2), ones_w, padding=pad).permute(0, 2, 3, 1) > 0
    reach_dx = torch.nn.grad.conv2d_input(ix.permute(0, 3, 1, 2).shape, ones_w, ig.permute(0, 3, 1, 2),
                                          padding=pad).permute(0, 2, 3, 1) > 0
    dw_mask = lambda a, gg: torch.nn.grad.conv2d_weight(a.permute(0, 3, 1, 2), ones_w.shape, gg.permute(0, 3, 1, 2),
                                                         padding=pad).permute(2, 3, 1, 0) > 0
    # a grad_out entry is in the weight-gradient sum of every tap, every cin, its cout -- taps that read padding
    # included (0 * NaN, as in IEEE arithmetic on the zero-padded sum)
    reach_dk = dw_mask(ix, torch.ones_like(ig))
    reach_dk[..., pg[3]] = True
    for got, reach, what in ((out, reach_out, 'forward'), (dx, reach_dx, 'grad_x'), (dk, reach_dk, 'grad_kernel')):
        assert torch.equal(torch.isnan(got), reach), f'{name} {what}: NaN set differs from the outputs that sum it'


def test_rejects_what_it_cannot_take():
    L = _lib()
    need = ctypes.c_size_t()
    with pytest.raises(RuntimeError, match='bad shape'):
        L.call('conv_tc_forward', 'cuda', None, None, None, 1, 8, 8, 8, 3, 3, 16, None, None, None, ctypes.byref(need))
    with pytest.raises(RuntimeError, match='bad shape'):
        L.call('conv_tc_forward', 'cuda', None, None, None, 1, 8, 8, 64, 2, 2, 16, None, None, None, ctypes.byref(need))
    x = torch.zeros((1, 8, 8, 64), device='cuda')
    k = torch.zeros((3, 3, 64, 16), device='cuda')
    b = torch.zeros(16, device='cuda')
    out = torch.empty((1, 8, 8, 16), device='cuda')
    planes = torch.empty(2 * 64 * 64, dtype=torch.float16, device='cuda')
    L.call('conv_tc_forward', 'cuda', None, None, None, 1, 8, 8, 64, 3, 3, 16, None, None, None, ctypes.byref(need))
    ws = L.workspace(need.value, 'cuda')
    with pytest.raises(RuntimeError, match='workspace'):
        L.call('conv_tc_forward', 'cuda', L.ptr(x), L.ptr(k), L.ptr(b), 1, 8, 8, 64, 3, 3, 16, L.ptr(out), L.ptr(planes),
               L.ptr(ws), ctypes.byref(ctypes.c_size_t(need.value - 1)))


# ------------------------------------------------------------------------------------------------ the training step
from test_gpu_train_state import L  # noqa: E402,F401  (the library fixture of the three-step test)


@pytest.fixture
def f16x2_step(monkeypatch):
    """RAFT.compile (and SmallRAFT's) defaults to train_precision='f16x2' for the test, and every _ConvTC application is
    counted, so that the existing step tests run unchanged on the tensor-core convolutions."""
    from tf_raft_b200 import model as M, train as Tr
    compile_, apply_ = M.RAFT.compile, Tr._ConvTC.apply
    calls = []
    monkeypatch.setattr(M.RAFT, 'compile', lambda self, *a, train_precision='f16x2', **kw:
                        compile_(self, *a, train_precision=train_precision, **kw))
    monkeypatch.setattr(Tr._ConvTC, 'apply', lambda *a: calls.append(1) or apply_(*a))
    return calls


@pytest.mark.parametrize('variant,shape,iters', [('small', (64, 96), 3), ('raft', (64, 96), 2)])
def test_f16x2_step_vs_oracle_autograd(f16x2_step, variant, shape, iters):
    """test_train.py::test_train_step_vs_oracle_autograd, its gates unchanged, on the f16x2 step: loss, global norm,
    every gradient, the whole gradient and every update."""
    import test_train
    test_train.test_train_step_vs_oracle_autograd(variant, shape, iters)
    assert f16x2_step, 'no convolution ran on the tensor cores'


@pytest.mark.parametrize('variant,iters', [('small', 3), ('raft', 2)])
def test_f16x2_three_train_steps_vs_oracle(f16x2_step, L, variant, iters):
    """test_gpu_train_state.py::test_three_train_steps_vs_oracle, its gates unchanged, on three f16x2 steps (m, v, t, the
    schedule and the moving statistics carried)."""
    import test_gpu_train_state
    test_gpu_train_state.test_three_train_steps_vs_oracle(L, variant, iters)
    assert f16x2_step, 'no convolution ran on the tensor cores'


def _unsup_grads(variant, train_precision):
    from tf_raft_b200 import RAFT, SmallRAFT
    from tf_raft_b200.losses import UnsupervisedLoss
    from tf_raft_b200.train import AdamW
    model = (RAFT if variant == 'raft' else SmallRAFT)(iters=3, seed=3)
    model.compile(optimizer=AdamW(weight_decay=1e-5, learning_rate=1e-4), clip_norm=1.0, loss=UnsupervisedLoss(),
                  train_precision=train_precision)
    gen = torch.Generator(device='cuda').manual_seed(0)
    im1 = torch.rand((2, 64, 96, 3), generator=gen, device='cuda') * 255
    im2 = torch.roll(im1, shifts=(2, 3), dims=(1, 2))
    logs = model.train_step((im1, im2))
    flat = model._trainer.flat
    return logs['loss'], {k: v.detach().clone() for k, v in flat.slot(flat.g).items()}


@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_f16x2_unsupervised_step_vs_fp32_step(variant):
    """One UnsupervisedLoss step, f16x2 against fp32: per tensor 5 % of its largest entry (+ the 2e-6 floor of
    test_train.py for biases in front of a norm layer), whole gradient 1e-2 relative L2."""
    loss32, g32 = _unsup_grads(variant, 'fp32')
    loss16, g16 = _unsup_grads(variant, 'f16x2')
    assert loss16 == pytest.approx(loss32, rel=1e-3)
    num = sum(float(((g16[k] - g32[k]) ** 2).sum()) for k in g32)
    den = sum(float((g32[k] ** 2).sum()) for k in g32)
    worst = max((float((g16[k] - g32[k]).abs().max()) / (5e-2 * float(g32[k].abs().max()) + 2e-6), k) for k in g32)
    print(f'{variant} unsupervised f16x2 vs fp32: relative L2 {math.sqrt(num / den):.3e}, worst per-tensor / gate '
          f'{worst[0]:.3f} ({worst[1]})')
    assert worst[0] <= 1.0, f'{worst[1]}: {worst[0]:.3f} x the per-tensor gate'
    assert math.sqrt(num / den) <= 1e-2, f'whole-gradient relative L2 {math.sqrt(num / den):.3e}'


def test_train_precision_is_validated():
    from tf_raft_b200 import RAFT
    from tf_raft_b200.train import AdamW
    model = RAFT(iters=2, seed=0)
    with pytest.raises(ValueError, match='train_precision'):
        model.compile(optimizer=AdamW(weight_decay=0.0), clip_norm=1.0, train_precision='f16')
