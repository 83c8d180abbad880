"""CPU checks of the mainloop sweep (tests/test_gpu_mainloop.py): the cases reach every corner of the shared wgmma
mainloop's configuration space that they claim to, judged by the geometry the library's own host code (tc_finalize,
tc_pick_tile) gives them through `conv_tc_probe describe`, and the fp64 model equals a direct triple loop."""
import itertools
import json
import os
import subprocess

import numpy as np
import pytest

import cases
import mainloop
import probe_build

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
PROBE_SRC = os.path.join(ROOT, 'tests', 'conv_tc_probe.cu')
TAPS = ((1, 1), (3, 3), (1, 5), (5, 1), (7, 7))
TILES = {(128, 1), (64, 2), (32, 4), (16, 8), (8, 16)}


@pytest.fixture(scope='module')
def described(tmp_path_factory):
    exe = probe_build.build(PROBE_SRC, 'raft_conv_tc_probe')
    if exe is None:
        pytest.skip('nvcc not found: the mainloop probe cannot be built')
    root = tmp_path_factory.mktemp('mainloop')
    plans = mainloop.mega_plans()
    all_cases = mainloop.sweep() + mainloop.epilogue_cases() + \
        [mainloop.mega_case(f'{n}_g{g}', p, 'mega', g) for n, p in plans.items() for g in mainloop.MEGA_GRIDS]
    out = {}
    for case in all_cases:
        d = root / case['name']
        d.mkdir()
        (d / 'case.txt').write_text(mainloop.build(case, 'a', 0)[0])
        res = subprocess.run([exe, 'describe', str(d)], capture_output=True, text=True, timeout=60)
        assert res.returncode == 0, res.stderr
        out[case['name']] = (case, json.loads(res.stdout)['layers'])
    return out


def _conv(described):
    """(spec layer, described layer, grid) of every sweep case."""
    names = {c['name'] for c in mainloop.sweep()}
    return [(c['layers'][0], d[0], c['grid'] or mainloop.SMS) for n, (c, d) in described.items() if n in names]


def test_describe_mirrors_the_spec(described):
    for case, layers in described.values():
        assert len(layers) == len(case['layers'])
        for l, d in zip(case['layers'], layers):
            assert d['total_chunks'] == mainloop.total_chunks(l)
            assert d['bn'] == l['bn'] and d['mma_n'] == mainloop.mma_n(l['bn']) and d['n_tiles_n'] == l['ntn']
            assert d['nstages'] == (l['nstages'] or mainloop.MAX_STAGES[l['bn']])
            B, hin, win, ho, wo = mainloop._geometry(l)[:5]
            assert (d['TW'], d['TH']) == cases.tc_tile(ho, wo)
            assert d['items'] == B * -(-ho // d['TH']) * -(-wo // d['TW']) * l['ntn']


def test_every_mma_width_at_every_ring_depth(described):
    got = {(d['bn'], d['nstages']) for _, d, _ in _conv(described)}
    want = {(bn, s) for bn, top in mainloop.MAX_STAGES.items() for s in range(2, top + 1)}
    assert want <= got, sorted(want - got)
    assert {mainloop.mma_n(bn) for bn, _ in got} == {16, 32, 64, 96, 128}


def test_column_tiles_taps_strides_and_segments(described):
    conv = _conv(described)
    assert {d['n_tiles_n'] for _, d, _ in conv} == {1, 2, 3}
    assert all(l['n_total'] % l['bn'] != 0 and (l['ntn'] - 1) * l['bn'] < l['n_total'] <= l['ntn'] * l['bn']
               for l, _, _ in conv)
    forms = {(l['taps'], l['stride'], len(l['segs'])) for l, d, _ in conv if not l['flatten']}
    assert forms == set(itertools.product(TAPS, (1, 2), (1, 2)))
    # stride 2 on odd and on even inputs, both ways
    s2 = {(l['img'][1] % 2, l['img'][2] % 2) for l, _, _ in conv if l['stride'] == 2}
    assert {0, 1} == {p[0] for p in s2} == {p[1] for p in s2}
    assert {d['chunks_per_tap'] for _, d, _ in conv} >= {1, 2, 3, 4, 5}
    segs = {l['segs'] for l, _, _ in conv if len(l['segs']) == 2}
    assert {(1, 3), (3, 1)} <= segs
    assert any(l['seg_c0'][1] > 0 for l, _, _ in conv if len(l['segs']) == 2)
    assert any(l['seg_c0'][0] > 0 for l, _, _ in conv)
    assert any(l['cinmap'] for l, _, _ in conv) and any(l['flatten'] for l, _, _ in conv)
    assert any(l['nw'] == 2 for l, _, _ in conv)


def test_chunks_against_ring_depth_and_group(described):
    ring, group = set(), set()
    for _, d, _ in _conv(described):
        t, s, g = d['total_chunks'], d['nstages'], d['group_chunks']
        ring.add('<' if t < s else '=' if t == s else '+1' if t == s + 1 else 'multiple' if t % s == 0 else 'other')
        assert d['total_mod_nstages'] == t % s and d['groups_per_tile'] == -(-t // g)
        group.add('1' if g == 1 and t > 2 else 'total-1' if g == t - 1 and g > 1 else 'total' if g == t else
                  'total+1' if g == t + 1 else 'between' if 1 < g < t - 1 else 'other')
    assert {'<', '=', '+1', 'multiple'} <= ring, ring
    assert {'1', 'between', 'total-1', 'total', 'total+1'} <= group, group
    assert {1, 2, 3, 5} <= {d['group_chunks'] for _, d, _ in _conv(described)}


def test_group_boundaries_land_on_every_ring_slot(described):
    """For every ring depth, the chunks that close a promotion group (the IEEE promotion follows their MMAs) fall on
    every ring slot, counted along CTA 0's walk across its tiles (the ring carries across tiles)."""
    slots = {}
    for _, d, grid in _conv(described):
        s, t, g = d['nstages'], d['total_chunks'], d['group_chunks']
        n_tiles = len(range(0, d['items'], grid))
        for k in range(n_tiles):
            for e in range(g, t + g, g):
                slots.setdefault(s, set()).add((k * t + min(e, t) - 1) % s)
    for s in range(2, 6):
        assert slots.get(s) == set(range(s)), (s, slots.get(s))


def test_grids_carry_the_ring_across_tiles(described):
    conv = _conv(described)
    for grid in (2, 3, 7, mainloop.SMS):                                # more tiles than CTAs, a ragged last round
        assert any(d['items'] > grid and d['items'] % grid for _, d, g in conv if g == grid), grid
    assert max(d['items'] for _, d, g in conv if g == 1) >= 20           # one CTA walks 20 tiles or more


def test_every_pixel_tile_on_ragged_images(described):
    ragged = set()
    for l, d, _ in _conv(described):
        ho, wo = mainloop._geometry(l)[3:5]
        if wo % d['TW'] and (d['TH'] == 1 or ho % d['TH']):
            ragged.add((d['TW'], d['TH']))
    assert ragged == TILES, ragged


def test_mega_plans_recarve_and_run_deep(described):
    carve = described['carve_g1'][1]
    sizes = [d['stage_bytes'] for d in carve]
    assert all(a != b for a, b in zip(sizes, sizes[1:])) and len(carve) >= 3
    assert carve[1]['nseg'] == 2 and (carve[2]['kh'], carve[2]['kw']) == (5, 1)
    assert carve[-1]['bn'] == 16 and carve[-1]['total_chunks'] == 1
    deep = described['deep_g1'][1]
    assert all(d['total_chunks'] == 1 and d['nstages'] == mainloop.MAX_STAGES[16] == 5 for d in deep)
    for name in described:
        if name.startswith(('carve_', 'deep_')):
            layers = described[name][1]
            assert sum(d['items'] for d in layers) > mainloop.SMS          # more items than CTAs at every grid
    # the item queue of update_mega_kernel must hold the producer's lead of nstages + 1 items (mega.cuh static_assert)
    with open(os.path.join(ROOT, 'tf_raft_b200', 'csrc', 'mega.cuh')) as f:
        assert 'static_assert(kMegaMaxStages + 1 < kMegaQueue' in f.read()


def test_epilogue_cases_at_two_widths(described):
    kinds = {}
    for c in mainloop.epilogue_cases():
        l = c['layers'][0]
        kinds.setdefault(l['epi'], set()).add(l['bn'])
    assert set(kinds) == {'linear', 'zr', 'q', 'advance'} and all(len(v) == 2 for v in kinds.values())


def _direct(a_hi, a_lo, seg_c0, chunks, geometry, w_hi, w_lo, inv, bias):
    B, hin, win, ho, wo, kh, kw, ph, pw, stride = geometry
    E = np.zeros((B, ho, wo, w_hi.shape[1]))
    S = np.zeros_like(E)
    for b, y, x, n in itertools.product(range(B), range(ho), range(wo), range(w_hi.shape[1])):
        e = s = 0.0
        for ty, tx in itertools.product(range(kh), range(kw)):
            iy, ix = y * stride + ty - ph, x * stride + tx - pw
            if not (0 <= iy < hin and 0 <= ix < win):
                continue
            k = 0
            for seg, (c0, ch) in enumerate(zip(seg_c0, chunks)):
                for c in range(c0, c0 + 64 * ch):
                    ah, al = float(a_hi[seg][b, iy, ix, c]), float(a_lo[seg][b, iy, ix, c])
                    wh, wl = float(w_hi[ty * kw + tx, n, k]), float(w_lo[ty * kw + tx, n, k])
                    e += ah * wh + ah * wl + al * wh
                    s += abs(ah * wh) + abs(ah * wl) + abs(al * wh)
                    k += 1
        E[b, y, x, n] = e * inv + float(bias[n])
        S[b, y, x, n] = s * inv + abs(float(bias[n]))
    return E.reshape(-1, E.shape[-1]), S.reshape(-1, S.shape[-1])


@pytest.mark.parametrize('stride', (1, 2))
def test_model_equals_direct_triple_loop(stride):
    """The im2col model on two segments (one read from channel 64), a 3 x 2 tap window and odd sizes equals a direct
    fp64 triple loop over pixels, taps and channels, zero padding included."""
    rng = np.random.default_rng(5)
    B, hin, win, kh, kw = 2, 5, 4, 3, 2
    ho, wo = mainloop.out_hw(hin, win, stride)
    ph, pw = mainloop.same_pads(kh, hin, ho, stride), mainloop.same_pads(kw, win, wo, stride)
    seg_c0, chunks = (0, 64), (1, 1)
    a = [rng.standard_normal((B, hin, win, 64)).astype(np.float32),
         rng.standard_normal((B, hin, win, 128)).astype(np.float32)]
    a_hi, a_lo = zip(*(cases.split_f16(x) for x in a))
    w_hi, w_lo = cases.split_f16(rng.standard_normal((kh * kw, 5, 128)).astype(np.float32) * 4096)
    bias = rng.standard_normal(5).astype(np.float32)
    geometry = (B, hin, win, ho, wo, kh, kw, ph, pw, stride)
    E, S = mainloop.model(a_hi, a_lo, seg_c0, chunks, geometry, w_hi, w_lo, 2.0 ** -12, bias)
    E2, S2 = _direct(a_hi, a_lo, seg_c0, chunks, geometry, w_hi, w_lo, 2.0 ** -12, bias)
    np.testing.assert_allclose(E, E2, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(S, S2, rtol=1e-12, atol=1e-12)


def test_packed_expectation_places_ranges_and_flattens():
    rng = np.random.default_rng(6)
    w = rng.standard_normal((3, 3, 10, 4)).astype(np.float32)
    hi, lo, s, _ = mainloop.packed_expected([w], 64, 16, (2, 0, 6, 0, 6, 4, 32), False)
    assert hi.shape == (9, 16, 64) and 2 ** 12 <= np.abs(w).max() * s < 2 ** 13
    back = hi.astype(np.float64) + lo.astype(np.float64)
    np.testing.assert_allclose(back[:, :4, :6], np.transpose(w.reshape(9, 10, 4), (0, 2, 1))[:, :, :6] * s, rtol=2 ** -21)
    np.testing.assert_allclose(back[:, :4, 32:36], np.transpose(w.reshape(9, 10, 4), (0, 2, 1))[:, :, 6:] * s,
                               rtol=2 ** -21)
    assert not back[:, :4, 6:32].any() and not back[:, :4, 36:].any() and not back[:, 4:].any()
    hi, lo, s, _ = mainloop.packed_expected([w[..., :2], w[..., 2:]], 128, 16, None, True)
    assert hi.shape == (1, 16, 128)
    np.testing.assert_array_equal(hi[0, :4, :90], cases.split_f16(w.reshape(90, 4).T * np.float32(s))[0])
