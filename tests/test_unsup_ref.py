"""The self-supervised loss without a GPU: the restatement (oracle/unsup_np.py) on known answers, and the bidirectional
training graph plus UnsupervisedLoss, with the CUDA pieces replaced by CPU stand-ins, against the oracle's loss and its
torch.autograd gradient for every trainable variable."""
import numpy as np
import pytest
import torch

import cases
from oracle import occlusion_np, raft_torch as rt, unsup_np, weights

GAMMA = 0.8


def _texture(b, h, w, seed):
    return np.random.default_rng(seed).uniform(0, 255, (b, h, w, 3)).astype(np.float32)


def test_census_offsets_and_constant_image():
    """48 offsets of the 7 x 7 window in row-major order; a constant image has census 0 wherever the window lies inside
    the frame, and not at the border, where the frame is padded with grey 0."""
    assert len(unsup_np.OFFSETS) == 48 and unsup_np.OFFSETS[0] == (-3, -3) and unsup_np.OFFSETS[24] == (0, 1)
    c = unsup_np.census(np.full((2, 12, 15, 3), 97.0, dtype=np.float32))
    assert c.shape == (2, 12, 15, 48) and c.dtype == np.float32
    assert not c[:, 3:-3, 3:-3].any()
    assert c[:, 0, 0].min() < 0 and (c[:, :3] != 0).any(axis=-1).all()


def test_census_channel_is_the_neighbour_difference():
    """One channel worked by hand: offset (dy, dx) = (1, -2) at (y, x) = (4, 5)."""
    im = _texture(1, 9, 11, 1)
    g = unsup_np.grey(im)
    k = unsup_np.OFFSETS.index((1, -2))
    t = np.float32(g[0, 5, 3] - g[0, 4, 5])
    assert unsup_np.census(im)[0, 4, 5, k] == t / np.sqrt(np.float32(0.81) + t * t)


@pytest.mark.parametrize('n', [1, 4])
def test_identical_images_with_zero_flow_give_the_floor_of_the_penalty(n):
    """D = 0 everywhere, nothing occluded: every masked pixel costs 0.01^0.4, so L_c = 0.01^0.4 sum_i gamma^(n-1-i); the
    zero flow has no smoothness cost."""
    im = _texture(2, 16, 20, 2)
    zero = [torch.zeros((2, 16, 20, 2), dtype=torch.float64, requires_grad=True) for _ in range(n)]
    with torch.no_grad():
        total, fw, bw = unsup_np.loss(im, im, zero, zero, return_terms=True)
    want = 0.01 ** 0.4 * sum(GAMMA ** (n - 1 - i) for i in range(n))
    for lc, ls in (fw, bw):
        assert float(lc) == pytest.approx(want, rel=1e-13)
        assert float(ls) == 0.0
    assert float(total) == pytest.approx(want, rel=1e-13)


def test_integer_shift_with_the_exact_flow_has_zero_distance():
    """image2 is image1 moved by (3, 2) px: with the flow (3, 2) every masked pixel whose source census window lies
    inside the frame lands on an integer texel with the same census, D = 0 exactly; the backward flow (-3, -2) likewise."""
    b, h, w = 2, 20, 26
    im1 = _texture(b, h, w, 3)
    im2 = _texture(b, h, w, 4)
    im2[:, 2:, 3:] = im1[:, :-2, :-3]
    fw = torch.zeros((b, h, w, 2), dtype=torch.float64)
    fw[..., 0], fw[..., 1] = 3.0, 2.0
    bw = -fw
    occ_fw, occ_bw = occlusion_np.fb_occlusion(fw.float().numpy(), bw.float().numpy())
    c1, c2 = unsup_np.census(im1), unsup_np.census(im2)
    border = unsup_np.border_mask(b, h, w)
    checked = 0
    for ct, cs, flow, occ, (sx, sy) in ((c1, c2, fw, occ_fw, (3, 2)), (c2, c1, bw, occ_bw, (-3, -2))):
        D, inside = unsup_np.distance(torch.from_numpy(ct).double(), torch.from_numpy(cs).double(), flow)
        ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing='ij')
        src_inside = (xs + sx >= 3) & (xs + sx <= w - 4) & (ys + sy >= 3) & (ys + sy <= h - 4)
        sel = border & ~occ & src_inside[None]
        assert sel.sum() > 100 and bool(inside.numpy()[sel].all())
        assert not D.numpy()[sel].any()
        assert D.numpy()[border & ~sel].max() > 0                     # the rest of the frame is not trivially zero
        checked += int(sel.sum())
    assert checked > 500


def test_constant_flow_has_zero_smoothness():
    im = torch.from_numpy(_texture(2, 10, 13, 5)).double()
    flow = torch.empty((2, 10, 13, 2), dtype=torch.float64)
    flow[..., 0], flow[..., 1] = -4.25, 7.5
    assert float(unsup_np.smoothness(im, flow, 150.0)) == 0.0
    flow[:, :, 6:, 0] += 1.0                                           # one vertical edge: horizontal pairs only
    s = float(unsup_np.smoothness(im, flow, 150.0))
    assert s > 0


def test_smoothness_edge_weight_known_answer():
    """2 x 2 image, one flow step of (1, -2) between the columns: each horizontal pair costs w * 3 / 2 with
    w = exp(-150 * mean_c |dI| / 255); the vertical pairs cost nothing."""
    im = torch.tensor([[[[0, 0, 0], [51, 102, 0]], [[0, 0, 0], [0, 0, 0]]]], dtype=torch.float64)
    flow = torch.zeros((1, 2, 2, 2), dtype=torch.float64)
    flow[:, :, 1, 0], flow[:, :, 1, 1] = 1.0, -2.0
    w_top, w_bottom = np.exp(-150 * 51 / 255), 1.0
    want = ((w_top + w_bottom) * 1.5 / 2 + 0.0) / 2
    assert float(unsup_np.smoothness(im, flow, 150.0)) == pytest.approx(want, rel=1e-14)


def test_loss_arguments_are_checked():
    from tf_raft_b200 import UnsupervisedLoss
    assert UnsupervisedLoss().smoothness_weight == 0.5 and UnsupervisedLoss().edge_weight == 150.0
    for bad in (dict(census_weight=-1.0), dict(gamma=float('nan')), dict(alpha2=float('inf'))):
        with pytest.raises(ValueError):
            UnsupervisedLoss(**bad)


# --------------------------------------------------------------------------------------------- graph + loss on the CPU
class _CpuLookup:
    @staticmethod
    def apply(coords, radius, *pyr):
        cb = rt.CorrBlock.__new__(rt.CorrBlock)
        cb.corr_pyramid, cb.num_levels, cb.radius = list(pyr), len(pyr), radius
        return cb.retrieve(coords)


class _CpuCorrBlock:
    def __init__(self, f1, f2, num_levels=4, radius=4, precision=None):
        self.corr_pyramid = [p.contiguous() for p in rt.CorrBlock(f1, f2, num_levels, radius).corr_pyramid]


class _CpuUnsupLoss:
    """The autograd function's contract, restated by the oracle in float64: (2n, B, H, W, 2) flows, [image1; image2]
    census, images and occlusion."""
    @staticmethod
    def apply(flows, census, images, occ, census_weight, smoothness_weight, edge_weight, gamma):
        n, b = flows.shape[0] // 2, flows.shape[1]
        mask = torch.from_numpy(unsup_np.border_mask(2 * b, *flows.shape[2:4])) & ~occ
        fw = unsup_np.direction_terms(census[:b], census[b:], images[:b], mask[:b], list(flows[:n]), gamma, edge_weight)
        bw = unsup_np.direction_terms(census[b:], census[:b], images[b:], mask[b:], list(flows[n:]), gamma, edge_weight)
        return (census_weight * (fw[0] + bw[0]) / 2 + smoothness_weight * (fw[1] + bw[1]) / 2).float()


def _cpu_occlusion(flow_fw, flow_bw, alpha1=0.01, alpha2=0.5):
    return tuple(torch.from_numpy(o) for o in occlusion_np.fb_occlusion(flow_fw.numpy(), flow_bw.numpy(), alpha1, alpha2))


@pytest.mark.parametrize('variant,iters', [('small', 3), ('raft', 2)])
def test_bidirectional_graph_and_loss_match_oracle_autograd_on_cpu(monkeypatch, variant, iters):
    """TrainGraph.forward_bidirectional + UnsupervisedLoss, the CUDA pieces replaced by CPU stand-ins (lookup, correlation
    forward, census, occlusion and the loss function by the oracle), against the oracle forward on the batch-2B pair
    ([image1; image2], [image2; image1]) -- the same fnet / cnet batches, cnet's BatchNorm over 2B images -- and the
    float64 loss: the same loss and the same torch.autograd gradient for every trainable variable."""
    import tf_raft_b200.losses as L
    import tf_raft_b200.train as tr
    monkeypatch.setattr(tr, '_Lookup', _CpuLookup)
    monkeypatch.setattr(tr, 'CorrBlock', _CpuCorrBlock)
    monkeypatch.setattr(tr, '_UnsupLoss', _CpuUnsupLoss)
    monkeypatch.setattr(L, 'census_transform', lambda im: torch.from_numpy(unsup_np.census(im.numpy())))
    monkeypatch.setattr(L, 'fb_occlusion', _cpu_occlusion)
    p = weights.init_params(variant, 21, bias_scale=0.05, norm_jitter=0.1)
    im1, im2 = cases.images(2, 64, 96, 3, 4)
    frozen = ('moving_mean', 'moving_variance')
    leaves = {k: torch.tensor(v, dtype=torch.float32, requires_grad=not k.endswith(frozen)) for k, v in p.items()}
    names = [k for k, v in leaves.items() if v.requires_grad]
    preds_o = rt.forward(leaves, np.concatenate([im1, im2]), np.concatenate([im2, im1]), variant, iters, training=True)
    loss_o = unsup_np.loss(im1, im2, [q[:2] for q in preds_o], [q[2:] for q in preds_o])
    g_o = dict(zip(names, torch.autograd.grad(loss_o, [leaves[k] for k in names])))
    P = {k: torch.tensor(v, dtype=torch.float32, requires_grad=not k.endswith(frozen)) for k, v in p.items()}
    moving = {k: v.detach().clone() for k, v in P.items() if k.endswith(frozen)}
    graph = tr.TrainGraph(P, variant, 'fp32', moving)
    t1, t2 = torch.from_numpy(im1), torch.from_numpy(im2)
    preds = graph.forward_bidirectional(t1, t2, iters)
    assert len(preds[0]) == len(preds[1]) == iters and preds[0][0].shape == (2, 64, 96, 2)
    loss = L.UnsupervisedLoss()((t1, t2), preds)
    assert float(loss) == pytest.approx(float(loss_o), rel=1e-5)
    g_t = dict(zip(names, torch.autograd.grad(loss, [P[k] for k in names])))
    # The census sample is piecewise in the landing (floor picks the corners): a landing within fp32 rounding of a texel
    # boundary takes the other side's corners on one of the two forwards, which moves a variable's gradient by a few
    # 1e-4 of its largest entry (RAFT at this seed: one variable at 4e-4, every other below 5e-5).  Hence 1e-3 per
    # variable, and the whole gradient to 1e-4 in relative L2 norm.
    num = den = 0.0
    for k in names:
        tol = 1e-3 * float(g_o[k].abs().max()) + 2e-6
        assert float((g_t[k] - g_o[k]).abs().max()) <= tol, k
        num += float(((g_t[k] - g_o[k]).double() ** 2).sum())
        den += float((g_o[k].double() ** 2).sum())
    assert (num / den) ** 0.5 <= 1e-4
    if variant == 'raft':        # cnet's BatchNorm saw 2B images: its moving statistics moved
        assert any(float((moving[k] - P[k]).abs().max()) > 0 for k in moving if k.startswith('cnet.'))


# --------------------------------------------------------------------------------------------- the closed form
def _closed_vs_autograd(b, h, w, n, case='random', occ_p=0.3, seed=0, chunk=97, **kw):
    """unsup_np.direction_closed_form against torch.autograd of direction_terms on the same direction: L_c, L_s and
    every gradient element to 1e-12 relative (of the largest gradient entry).  chunk=97 makes the census chunks and the
    smoothness row bands small, so their seams fall everywhere."""
    from test_gpu_unsup import _flows, _texture
    cw, sw = kw.get('census_weight', 1.0), kw.get('smoothness_weight', 0.5)
    gamma, ew, norm = kw.get('gamma', GAMMA), kw.get('edge_weight', 150.0), kw.get('census_norm')
    rng = np.random.default_rng(seed)
    im_t, im_s = _texture(b, h, w, seed + 1), _texture(b, h, w, seed + 2)
    ct, cs = unsup_np.census(im_t), unsup_np.census(im_s)
    mask = unsup_np.border_mask(b, h, w) & (rng.random((b, h, w)) >= occ_p)
    flows = _flows(case, n, b, h, w, rng)
    leaves = [torch.from_numpy(f).double().requires_grad_(True) for f in flows]
    lc, ls = unsup_np.direction_terms(ct, cs, im_t, mask, leaves, gamma, ew, norm)
    want_g = [g.numpy() for g in torch.autograd.grad(cw / 2 * lc + sw / 2 * ls, leaves)]
    got_lc, got_ls, count, got_g = unsup_np.direction_closed_form(ct, cs, im_t, mask, flows, cw, sw, ew, gamma, norm,
                                                                  chunk=chunk)
    assert count == int(mask.sum())
    for got, want in ((got_lc, float(lc.detach())), (got_ls, float(ls.detach()))):
        if np.isnan(want):
            assert np.isnan(got)
        else:
            assert got == pytest.approx(want, rel=1e-12, abs=1e-300), (got, want)
    finite = [np.isfinite(g) for g in want_g]
    scale = max([float(np.abs(g[m]).max()) for g, m in zip(want_g, finite) if m.any()] + [0.0])
    for i, (g, wg, m) in enumerate(zip(got_g, want_g, finite)):
        np.testing.assert_array_equal(np.isfinite(g), m, err_msg=f'prediction {i}: non-finite pattern')
        assert float(np.abs(g[m] - wg[m]).max(initial=0.0)) <= 1e-12 * scale, f'prediction {i}'
    return count, got_lc, got_ls, got_g


@pytest.mark.parametrize('case', ['random', 'integer', 'leaving', 'flat', 'nonfinite'])
def test_closed_form_matches_autograd_on_every_flow_kind(case):
    _closed_vs_autograd(2, 24, 40, 3, case, seed=len(case))


@pytest.mark.parametrize('shape', [(3, 7, 7, 2), (2, 6, 40, 3), (2, 40, 6, 3), (1, 2, 2, 1), (5, 37, 53, 4)],
                         ids=['7x7', 'H<7', 'W<7', '2x2', 'ragged'])
def test_closed_form_matches_autograd_at_edge_shapes(shape):
    b, h, w, n = shape
    count = _closed_vs_autograd(b, h, w, n, occ_p=0.0 if h == 7 else 0.3)[0]
    if h == w == 7:
        assert count == b                                             # one masked pixel, (3, 3), per image
    if min(h, w) < 7:
        assert count == 0


@pytest.mark.parametrize('kw', [dict(gamma=0.0), dict(gamma=1.0), dict(gamma=1.25), dict(edge_weight=0.0),
                                dict(edge_weight=1e4), dict(census_weight=0.0), dict(smoothness_weight=0.0),
                                dict(census_norm=777.5), dict(occ_p=1.0), dict(occ_p=0.0)],
                         ids=lambda kw: '-'.join(f'{k}={v}' for k, v in kw.items()))
def test_closed_form_matches_autograd_at_parameter_edges(kw):
    kw = dict(kw)
    occ_p = kw.pop('occ_p', 0.3)
    count, lc, ls, grads = _closed_vs_autograd(2, 19, 31, 3, occ_p=occ_p, **kw)
    if occ_p == 1.0:
        assert count == 0 and lc == 0.0
    if kw.get('gamma') == 0.0:                                          # only the last prediction carries weight
        assert all(not g.any() for g in grads[:-1]) and grads[-1].any()
