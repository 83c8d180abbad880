"""CPU checks of the geometry sweep's case lists and fp64 references (tests/test_gpu_geometry.py): the grids reach the
code paths they are meant to reach, and the references used as truth are right."""
import numpy as np
import torch

import cases
from oracle import corr_np, raft_torch as rt, weights

ALL_TILES = {(128, 1), (64, 2), (32, 4), (16, 8), (8, 16)}


def test_tile_mirror_known_answers():
    assert cases.tc_tile(56, 128) == (128, 1)      # Sintel (436 x 1024 padded to 448 x 1024)
    assert cases.tc_tile(56, 64) == (64, 2)        # FlyingChairs-size benchmark grid (448 x 512)
    assert cases.tc_tile(8, 8) == (16, 8)
    assert cases.tc_tile(8, 12) == (16, 8)
    for h in range(1, 70):
        for w in range(1, 140):
            tw, th = cases.tc_tile(h, w)
            assert tw * th == 128 and (tw, th) in ALL_TILES
            area = -(-w // tw) * tw * (-(-h // th) * th)
            for t in (128, 64, 32, 16, 8):                       # least padded area, the wider tile on a tie
                other = -(-w // t) * t * (-(-h // (128 // t)) * (128 // t))
                assert area < other or (area == other and tw >= t)


def test_tile_grids_reach_every_tile_shape():
    tiles = [cases.tc_tile(h, w) for _, h, w in cases.TILE_GRIDS]
    assert set(tiles) == ALL_TILES, tiles
    b, h, w = cases.TILE_GRIDS[-1]
    tw, th = cases.tc_tile(h, w)
    assert b * -(-h // th) * -(-w // tw) == 36          # pixel tiles per layer: with ~15 layers, several times 132 work items
    # the loop test needs a 4-level pyramid on the 128 x 1 grid
    assert min(cases.TILE_GRIDS[0][1:]) >> 3 >= 1


def test_lookup_grids_reach_every_kernel_form():
    for levels, grids in cases.LOOKUP_GRIDS.items():
        deepest = [cases.level_sizes(h, w, levels)[-1] for _, h, w in grids]
        assert all(min(s) >= 1 for s in deepest)
        assert any(1 in s for s in deepest), (levels, deepest)                 # a deepest level 1 wide or 1 high
    vec = [all(lw % 4 == 0 for _, lw in cases.level_sizes(h, w, 4)) for _, h, w in cases.LOOKUP_GRIDS[4]]
    assert sorted(vec) == [False, True]                                     # 128-bit and scalar window loads
    assert not any(w % 4 == 0 for _, _, w in cases.LOOKUP_GRIDS[4][:1])


def test_pyramid_cases_cover_levels_channels_and_odd_sizes():
    levels = {c[4] for c in cases.PYRAMID_CASES}
    assert {1, 2, 4, 5, 6} <= levels
    assert {64, 128, 192, 256} <= {c[3] for c in cases.PYRAMID_CASES}
    pow2 = {float(np.sqrt(c)).is_integer() and (int(np.sqrt(c)) & (int(np.sqrt(c)) - 1)) == 0 for c in (64, 128, 192, 256)}
    assert pow2 == {True, False}                                                # corr_mul and corr_div scalings
    for b, h, w, c, lv in cases.PYRAMID_CASES:
        assert (h * w) % 128 != 0 and c % 64 == 0
        assert min(min(s) for s in cases.level_sizes(h, w, lv)) >= 1
    assert any(all(lh % 2 and lw % 2 for lh, lw in cases.level_sizes(h, w, lv)) and lv > 4
               for b, h, w, c, lv in cases.PYRAMID_CASES)                    # odd at every level, generic path
    assert any(b == 3 for b, *_ in cases.PYRAMID_CASES)


def test_fp64_pyramid_matches_the_literal_numpy_restatement():
    """The fp64 truth of the pyramid test (raft_torch.CorrBlock on double features) is the reference's volume, pooled the
    reference's way: it agrees with the op-by-op NumPy restatement to fp32 rounding, on odd sizes through 5 levels."""
    b, h, w, c, levels = 1, 31, 33, 64, 5
    f1, f2 = cases.fmaps(b, h, w, c, seed=3)
    truth = rt.CorrBlock(torch.from_numpy(f1).double(), torch.from_numpy(f2).double(), levels, 4).corr_pyramid
    lit = corr_np.CorrBlock(f1, f2, levels, 4).corr_pyramid
    for l, (lh, lw) in enumerate(cases.level_sizes(h, w, levels)):
        assert truth[l].shape == lit[l].shape == (b * h * w, lh, lw, 1)
        np.testing.assert_allclose(truth[l].numpy(), lit[l], atol=5e-6, rtol=1e-5)


def test_fp64_lookup_gradient_matches_finite_differences():
    """The backward truth (torch.autograd through raft_torch's sampler in fp64) is the derivative of the sampler, checked
    by central differences at non-integer coordinates, out-of-range ones (clamped: zero gradient) included."""
    b, h, w, levels, r = 1, 5, 7, 3, 2
    f1, f2 = cases.fmaps(b, h, w, 64, seed=4)
    pyr = [p.clone().requires_grad_(True)
           for p in rt.CorrBlock(torch.from_numpy(f1).double(), torch.from_numpy(f2).double(), levels, r).corr_pyramid]
    coords = torch.from_numpy(cases.lookup_coords(b, h, w, 'jitter', seed=8)).double().requires_grad_(True)

    def f(c, *p):
        cb = rt.CorrBlock.__new__(rt.CorrBlock)
        cb.corr_pyramid, cb.num_levels, cb.radius = list(p), levels, r
        return cb.retrieve(c)
    assert torch.autograd.gradcheck(f, (coords, *pyr), eps=1e-7, atol=1e-6)


def test_encoder_params_fit_both_encoders_and_every_norm():
    from tf_raft_b200.layers.extractor import BasicEncoder, SmallEncoder
    for variant, cls, out_dim in (('raft', BasicEncoder, 256), ('small', SmallEncoder, 128)):
        for norm in ('instance', 'batch', None):
            p = cases.encoder_params(variant, norm, out_dim)
            enc = cls(output_dim=out_dim, norm_type=norm, device='cpu')
            assert set(enc.params) == {k[len('enc.'):] for k in p}
            enc.load_params(p, 'enc.')
    # the refactored parameter generator draws the same values as before
    p = weights.init_params('small', 1234, bias_scale=0.05, norm_jitter=0.1)
    q = weights.draw_params(weights.param_shapes('small'), 1234, 0.05, 0.1)
    assert list(p) == list(q) and all(np.array_equal(p[k], q[k]) for k in p)


def test_encoder_plan_known_answers():
    """encoder_plan at the benchmark's 448 x 512: the stem and stage 1 on 224 x 256, stage 2 on 112 x 128 (the 128 x 1
    tile, whose stride-2 box is 256 elements wide), stage 3 on 56 x 64; even inputs pad the stride-2 3 x 3 convolutions
    after only."""
    plan = {e['name']: e for e in cases.encoder_plan(448, 512, 'raft')}
    assert len(plan) == 1 + 6 * 2 + 2 + 1
    assert [(e['hout'], e['wout'], e['tw'], e['th']) for e in (plan['stem'], plan['layer2.0.conv1'], plan['conv2'])] == \
        [(224, 256, 128, 1), (112, 128, 128, 1), (56, 64, 64, 2)]
    s2 = plan['layer2.0.conv1']
    assert (s2['stride'], s2['hin'], s2['win'], s2['pt'], s2['pl']) == (2, 224, 256, 0, 0)
    assert s2['tw'] * s2['stride'] == 256
    odd = {e['name']: e for e in cases.encoder_plan(70, 98, 'small')}['layer3.0.conv1']      # 18 x 25 -> 9 x 13
    assert (odd['hin'], odd['win'], odd['hout'], odd['wout'], odd['pt'], odd['pl']) == (18, 25, 9, 13, 0, 1)
    assert all(e['pt'] == e['pl'] == 0 for e in cases.encoder_plan(71, 99, 'raft') if e['k'] == 1)


def test_encoder_grids_reach_every_stride2_tile_and_parity():
    """Over every image with H in 8..400 and W in 8..1300, the stride-2 convolutions of the encoders reach 20
    combinations of (pixel tile, odd input height, odd input width) with an output of at least two tiles each way:
    five tiles times four parities.  ENCODER_GRIDS reaches all of them, and holds the smallest images.  The plan depends
    on the image only through the stem's output size, so one image per stem size is enumerated."""
    reach = {}
    for H in range(8, 401):
        for W in range(8, 1301):
            key = (-(-H // 2), -(-W // 2))
            if key not in reach:
                reach[key] = cases.stride2_combos(H, W, 'raft')
    universe = set().union(*reach.values())
    assert universe == {(tw, 128 // tw, oh, ow) for tw in (128, 64, 32, 16, 8) for oh in (0, 1) for ow in (0, 1)}
    for variant in ('raft', 'small'):
        got = set().union(*(cases.stride2_combos(H, W, variant) for H, W in cases.ENCODER_GRIDS))
        assert got == universe, sorted(universe - got)
    assert {(8, 8), (8, 9), (9, 8)} <= set(cases.ENCODER_GRIDS)
    last = cases.encoder_plan(8, 8, 'raft')[-1]
    assert (last['hin'], last['win']) == (1, 1)                      # stage 3 is one pixel: zero instance-norm variance


def test_fp64_encoder_output_shape_on_odd_sizes():
    """rt.encoder pads the stride-2 stages the TensorFlow way: the output is ceil(H / 8) x ceil(W / 8)."""
    p = cases.encoder_params('small', 'instance', 128)
    for H, W in ((70, 98), (36, 52)):
        x = torch.zeros(1, 3, H, W, dtype=torch.float64)
        out = rt.encoder(rt.Ops(p, torch.float64), x, 'enc', 'instance', False)
        assert tuple(out.shape) == (1, 128, -(-H // 8), -(-W // 8))


# ------------------------------------------------------------------------------------ large grids (test_gpu_large.py)
def test_lookup_path_mirror_known_answers():
    assert cases.lookup_path(1, 8, 32, 4, 4, 324) == 'window-vec'       # every level width a multiple of 4
    assert cases.lookup_path(2, 9, 13, 4, 3, 196) == 'window'
    assert cases.lookup_path(1, 8, 32, 4, 2, 100) == 'generic'          # no window kernel for radius 2
    assert cases.lookup_path(1, 17, 19, 5, 4, 405) == 'generic'         # ... nor for 5 levels
    assert cases.lookup_path(4, 56, 64, 4, 4, 384) == 'window-vec'      # the benchmark grid, the loop's operand planes
    assert cases.lookup_path(1, 180, 320, 4, 4, 324) == 'generic'       # 1440p: 3.3e9 level-0 elements
    assert cases.lookup_path(3, 136, 240, 4, 4, 324) == 'generic'       # 1080p padded to 1088, batch 3: 3.2e9


def test_large_cases_straddle_the_lookup_limits():
    """Each large case sits on the side of the 2^31 (and 2^32) element limits its comment gives, for RAFT (radius 4) and
    SmallRAFT (radius 3), with fp32 output rows (retrieve) and fp16 operand rows (the loop)."""
    expect = {(1, 215, 215): (2136750625, 'window'), (1, 216, 216): (2176782336, 'generic'),
              (41, 56, 128): (2106589184, 'window-vec'), (42, 56, 128): (2157969408, 'generic'),
              (1, 257, 256): (4328587264, 'generic')}
    assert cases.LARGE_CASES == tuple(expect)
    for (B, h, w), (elements, path) in expect.items():
        assert B * (h * w) ** 2 == elements
        assert (elements >= 2 ** 31) == (path == 'generic')
        for radius, strides in ((4, (324, 384)), (3, (196, 256))):
            for stride in strides:
                assert cases.lookup_path(B, h, w, 4, radius, stride) == path, (B, h, w, radius, stride)
    assert [B * (h * w) ** 2 > 2 ** 32 for B, h, w in cases.LARGE_CASES] == [False] * 4 + [True]


def test_large_samples_hold_the_boundary_queries():
    """The sampled queries of every large case: the first and last 4 of every image, and the queries whose level-0
    planes hold elements 2^31 and 2^32, with their neighbours."""
    want = {(1, 216, 216): [46028], (42, 56, 128): [299593], (1, 257, 256): [32640, 65280]}
    assert divmod(299593, 56 * 128) == (41, 44 * 128 + 73)              # image 41, pixel y = 44, x = 73
    for B, h, w in cases.LARGE_CASES:
        n = h * w
        bq = cases.boundary_queries(B, h, w)
        assert bq == want.get((B, h, w), [])
        qs = cases.large_sample(B, h, w)
        assert qs.dtype == np.int64 and np.all(np.diff(qs) > 0) and qs[0] == 0 and qs[-1] == B * n - 1
        s = set(qs.tolist())
        for q, e in zip(bq, (2 ** 31, 2 ** 32)):
            assert q * n <= e < (q + 1) * n
            assert {q - 1, q, q + 1} <= s
        for b in range(B):
            assert set(range(b * n, b * n + 4)) | set(range((b + 1) * n - 4, (b + 1) * n)) <= s
        assert len(s) >= 8 * B + 3 * len(bq) + 24                          # ~32 random queries besides
    np.testing.assert_array_equal(cases.large_sample(1, 216, 216), cases.large_sample(1, 216, 216))


def test_corr_rows_equal_the_oracle_pyramid_rows():
    """The subset reference of test_gpu_large.py equals the rows of oracle.raft_torch.CorrBlock in float64."""
    B, h, w, c = 3, 11, 13, 64
    f1, f2 = cases.fmaps(B, h, w, c, seed=3)
    full = rt.CorrBlock(torch.from_numpy(f1).double(), torch.from_numpy(f2).double(), 4, 4).corr_pyramid
    qs = np.array([0, 5, 142, 143, 300, 428])
    rows = cases.corr_rows(f1, f2, qs, 4)
    assert len(rows) == 4
    for l in range(4):
        assert rows[l].dtype == torch.float64 and rows[l].shape == full[l][qs].shape
        np.testing.assert_allclose(rows[l].numpy(), full[l][qs].numpy(), rtol=1e-13, atol=1e-13)
