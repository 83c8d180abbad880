"""The shared wgmma mainloop on its own (conv_tc.cuh: ring_acquire / ring_mma, tc_produce_tile / tc_consume_tile,
with_mma_n; mega.cuh: the work queue and the ring re-carve), against an fp64 model of its split arithmetic.

tests/conv_tc_probe.cu runs conv_tc_kernel, or a plan of layers in one update_mega_kernel launch, with the ring depth,
the promotion group and the grid set by the case (tests/mainloop.py: the covering design, checked on the CPU by
tests/test_mainloop_cases.py), and dumps the exact fp16 operands the MMAs read.  From them mainloop.model gives E (the
split arithmetic, exact in fp64) and S (its magnitude) per output.  Three data kinds:

a. Small integers (activations in [-8, 8], weights in [-7, 7], bias 0): every operand is an exact fp16 value with
   lo = 0, and sum |a||w| stays below 2^24 in units of the smallest non-zero product (asserted), so every partial sum is
   exact in fp32 whatever the summation order or the tensor core's rounding: every output equals E bit for bit.  Dense
   data catches a wrong tap offset, chunk, segment, seg_c0, column tile, pixel tile, stride, padding or swizzle at
   every output.
b. Positive operands with lo != 0: nothing cancels, so S ~ |E| and a relative defect cannot hide.
c. Mixed-sign N(0, 1) operands; also compared with fp64 of the unsplit fp32 operands.

The bound for b and c, |got - E| <= 2u (12 g + n_groups + 2) S with u = 2^-24 and g = min(group_chunks, chunks per
tile): a promotion group is a chain of 12 g MMA steps (three k16 passes, hi.hi hi.lo lo.hi, over four k16 slices per
chunk) into one fp32 accumulator; each step may lose 2u of the running |sum| <= S (the tensor core's accumulation is not
round-to-nearest: 2u where IEEE addition would lose u); each of the n_groups IEEE promotions loses u <= 2u; the epilogue's
exact 2^-k scaling and its bias add lose at most 2u S more.  A dropped hi.lo or lo.hi pass moves an output by about
2^-11 relative, a group that is never promoted drops whole chunks, a slot read one phase late reads another chunk: all
far outside the bound.  Activations add the fast sigmoid / tanh error (__expf, __fdividef: ~1e-7, conv_tc.cuh:107-108),
taken here as ACT = 1e-6.

Side checks on every run: the hi/lo output planes equal cases.split_f16 of the fp32 result bit for bit; every canary
outside the written columns, and every fp32 row past the last pixel, is untouched; the packed weight planes equal
split_f16(w 2^k) in the [tap][cout_pad][cin_pad] layout with zero padding and the TcCinMap ranges in place.

update_mega_kernel: synthetic plans (mainloop.mega_plans) at grids 1, 2, 3, 7 and one CTA per SM equal, bit for bit,
the same layers run one conv_tc_kernel launch each, and that per-layer run passes the model checks.
"""
import json
import os
import subprocess

import numpy as np
import pytest

import cases
import mainloop
import probe_build

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
PROBE_SRC = os.path.join(ROOT, 'tests', 'conv_tc_probe.cu')
U = mainloop.U
ACT = 1e-6
WORST = {}

SWEEP = [(c, k) for c in mainloop.sweep() for k in 'abc']
EPILOGUES = [(c, k) for c in mainloop.epilogue_cases() for k in 'bc']
PLANS = [(n, k) for n in mainloop.mega_plans() for k in ('bc' if n == 'carve' else 'c')]


def _seed(name, kind):
    return sum(map(ord, name + kind)) * 7919 % 100003


@pytest.fixture(scope='module')
def runs(tmp_path_factory):
    """Every case written, then run in one probe process; {(name, kind): (case, meta, described layers)}."""
    exe = probe_build.build(PROBE_SRC, 'raft_conv_tc_probe')
    assert exe is not None, 'nvcc not found'
    root = str(tmp_path_factory.mktemp('mainloop_gpu'))
    todo = [(c, k, _seed(c['name'], k)) for c, k in SWEEP + EPILOGUES]
    for name, kind in PLANS:
        plan = mainloop.mega_plans()[name]
        todo.append((mainloop.mega_case(f'{name}_conv', plan, 'conv', 0), kind, _seed(name, kind)))
        todo += [(mainloop.mega_case(f'{name}_g{g}', plan, 'mega', g), kind, _seed(name, kind)) for g in mainloop.MEGA_GRIDS]
    built = {}
    for case, kind, seed in todo:
        _, meta = mainloop.build(case, kind, seed, root)
        built[(case['name'], kind)] = (case, meta)
    dirs = [m['dir'] for _, m in built.values()]
    res = subprocess.run([exe, 'run'] + dirs, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr
    dec, text, pos, desc = json.JSONDecoder(), res.stdout, 0, {}
    while True:
        while pos < len(text) and text[pos].isspace():
            pos += 1
        if pos >= len(text):
            break
        doc, pos = dec.raw_decode(text, pos)
        desc[doc['case']] = doc['layers']
    out = {key: (case, meta, desc[meta['dir']]) for key, (case, meta) in built.items()}
    yield out
    for kind in sorted(WORST):
        print(f'\nmainloop: worst |got - E| / bound, kind {kind}: {WORST[kind][0]:.4f} ({WORST[kind][1]})')


def _u16(path, shape):
    return np.fromfile(path, dtype=np.uint16).reshape(shape)


def _f32(path):
    return np.fromfile(path, dtype=np.float32)


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def _ratio(kind, name, err, tol):
    r = float((err / np.maximum(tol, 1e-300)).max()) if err.size else 0.0
    if r > WORST.get(kind, (0.0, ''))[0]:
        WORST[kind] = (r, name)
    return r


def check_case(case, meta, layers_desc, label):
    """Every check of one probe run.  Returns the worst |got - E| / bound."""
    d, kind = meta['dir'], meta['kind']
    planes = []
    for i, P in enumerate(meta['planes']):
        shape = (P['B'], P['H'], P['W'], P['cs'])
        hi, lo = _u16(f'{d}/P{i}_hi.bin', shape), _u16(f'{d}/P{i}_lo.bin', shape)
        if P['data'] is not None:                            # split_plane_kernel: the NumPy split, bit for bit
            eh, el = cases.split_f16(P['data'])
            assert np.array_equal(hi, eh.view(np.uint16)) and np.array_equal(lo, el.view(np.uint16)), f'plane {i}'
        planes.append((hi, lo))
    bufs = [_f32(f'{d}/B{i}.bin') for i in range(len(meta['bufs']))]
    written16 = {i: np.zeros(meta['planes'][i]['cs'], bool) for i in range(len(planes))}
    worst = 0.0
    for li, (m, desc) in enumerate(zip(meta['layers'], layers_desc)):
        l = m['spec']
        B, hin, win, ho, wo, kh, kw, ph, pw = m['geometry']
        npix, n_total, bn, ntn = m['npix'], l['n_total'], l['bn'], l['ntn']
        taps = kh * kw
        where = f'{label} layer {li}'
        # ---- packed weights ----
        whi = _u16(f'{d}/L{li}_whi.bin', (taps, m['cout_pad'], m['cin_pad']))
        wlo = _u16(f'{d}/L{li}_wlo.bin', (taps, m['cout_pad'], m['cin_pad']))
        scale = _f32(f'{d}/L{li}_scale.bin')
        eh, el, s, full = mainloop.packed_expected(m['w'], m['cin_pad'], m['cout_pad'], m['cmap'], l['flatten'])
        assert scale[0] == s and scale[1] == 1.0 / s, (where, scale, s)
        assert np.array_equal(whi, eh.view(np.uint16)) and np.array_equal(wlo, el.view(np.uint16)), where
        # ---- model ----
        a_hi = [mainloop.f16(planes[p][0]) for p in m['seg_planes']]
        a_lo = [mainloop.f16(planes[p][1]) for p in m['seg_planes']]
        bias = np.zeros(m['cout_pad'], np.float32)
        bias[:sum(b.size for b in m['b'])] = np.concatenate(m['b'])
        geometry = m['geometry'] + (l['stride'],)
        E, S = mainloop.model(a_hi, a_lo, l['seg_c0'], l['segs'], geometry, mainloop.f16(whi), mainloop.f16(wlo),
                              float(scale[1]), bias)
        tb = mainloop.bound(S, desc['total_chunks'], l['group'])
        if kind == 'a':
            assert not any(x.any() for x in a_lo) and not wlo.any(), where      # every operand exact: lo = 0
            assert S.max() < 2 ** 24, where                                      # every partial sum exact in fp32
        if kind == 'c' and all(meta['planes'][p]['data'] is not None for p in m['seg_planes']):
            a32 = [meta['planes'][p]['data'] for p in m['seg_planes']]
            T, _ = mainloop.model(a32, [np.zeros_like(x) for x in a32], l['seg_c0'], l['segs'], geometry,
                                  full * np.float32(s), np.zeros_like(full), float(scale[1]), bias)
        else:
            T = None

        def against(got, want, tol, cols, what):
            nonlocal worst
            err = np.abs(got.astype(np.float64) - want)
            if kind == 'a':
                bad = _bits(got) != _bits(want.astype(np.float32))
                assert not bad.any(), f'{where} {what}: {int(bad.sum())} outputs differ from the exact model'
                assert np.array_equal(want.astype(np.float32).astype(np.float64), want), where
            else:
                r = _ratio(kind, where, err, tol)
                worst = max(worst, r)
                assert r <= 1.0, f'{where} {what}: {int((err > tol).sum())} outputs off the model (worst {r:.2f} x bound)'

        mode, cols = m['mode'], slice(0, n_total)
        ext = 7
        want32 = None
        if mode == mainloop.EPI_LINEAR:
            v, tol = E[:, cols], tb[:, cols]
            if l['epi'] == 'linear':
                sc = bufs[m['post'][0]][:n_total].astype(np.float64)
                sh = bufs[m['post'][1]][:n_total].astype(np.float64)
                rb, rs, rc0 = m['residual']
                r = meta['bufs'][rb]['data'].reshape(-1, rs)[:npix, rc0:rc0 + n_total].astype(np.float64)
                v1 = v * sc + sh
                tol = np.abs(sc) * tol + 2 * U * (np.abs(v * sc) + np.abs(sh))
                v1 = np.maximum(v1, 0) * 0.25
                tol = tol * 0.25
                v = np.maximum(v1 + r, 0)
                tol = tol + 2 * U * (np.abs(v1) + np.abs(r))
            if 'out32' in m:
                ob, fs, fc0 = m['out32']
                o = bufs[ob].reshape(npix + ext, fs)
                got = o[:npix, fc0:fc0 + n_total]
                against(got, v, tol, cols, 'fp32 output')
                if T is not None and l['epi'] == 'plain':
                    err = np.abs(got - T[:, cols])
                    assert (err <= tb[:, cols] + 2.0 ** -21 * S[:, cols]).all(), f'{where}: off the unsplit fp64 product'
                canary = np.ones_like(o, bool)
                canary[:npix, fc0:fc0 + n_total] = False
                assert (o.view(np.uint32)[canary] == mainloop.CANARY32).all(), f'{where}: fp32 canary overwritten'
                want32 = np.zeros((npix, m['cout_pad']), np.float32)
                want32[:, :n_total] = got
            if l['epi'] == 'advance':
                cb, fb = m['adv']
                c_in = meta['bufs'][cb]['data'].reshape(npix, 2)
                c_out, flow = bufs[cb].reshape(npix, 2), bufs[fb].reshape(npix, 2)
                got = o[:npix, :2]
                assert np.array_equal(_bits(c_out), _bits(c_in + got)), f'{where}: coords1 += delta'
                yy, xx = np.meshgrid(np.arange(ho), np.arange(wo), indexing='ij')
                grid = np.tile(np.stack([xx, yy], -1).reshape(-1, 2), (B, 1)).astype(np.float32)
                assert np.array_equal(_bits(flow), _bits(c_out - grid)), f'{where}: flow = coords1 - grid'
            if 'out16' in m:
                pi, hc0 = m['out16']
                if want32 is None:
                    want32 = np.zeros((npix, m['cout_pad']), np.float32)
                if 'concat' in m:
                    cat = meta['bufs'][m['concat'][0]]['data'].reshape(npix, 2)
                    want32[:, n_total:n_total + 2] = cat
                hi, lo = (x.reshape(npix, -1) for x in planes[pi])
                if 'out32' not in m:                             # fp16 planes only: their value against the model
                    val = mainloop.f16(hi[:, hc0:hc0 + n_total]).astype(np.float64) + \
                        mainloop.f16(lo[:, hc0:hc0 + n_total]).astype(np.float64)
                    against(val, v, tol + 2.0 ** -21 * np.abs(v) + 2.0 ** -24, cols, 'fp16 planes')
                    eh, el = cases.split_f16(want32)            # columns past n_total: zeros (or concat), exactly
                    eh[:, :n_total] = mainloop.f16(hi[:, hc0:hc0 + n_total])
                    el[:, :n_total] = mainloop.f16(lo[:, hc0:hc0 + n_total])
                else:
                    eh, el = cases.split_f16(want32)
                for nt in range(ntn):
                    for c0 in range(0, bn, 32):
                        if bn - c0 < 32:
                            continue                             # a partial 32-column chunk writes no fp16 planes
                        c = nt * bn + c0
                        written16[pi][hc0 + c:hc0 + c + 32] = True
                        assert np.array_equal(hi[:, hc0 + c:hc0 + c + 32], eh[:, c:c + 32].view(np.uint16)), where
                        assert np.array_equal(lo[:, hc0 + c:hc0 + c + 32], el[:, c:c + 32].view(np.uint16)), where
        elif mode == mainloop.EPI_GRU_ZR:
            zb, hb, hid = m['gru']
            z = bufs[zb].reshape(npix, hid)
            sig = 1 / (1 + np.exp(-E[:, :2 * hid]))
            against(z, sig[:, :hid], 0.25 * tb[:, :hid] + ACT, slice(0, hid), 'z gate')
            h = meta['bufs'][hb]['data'].reshape(npix, hid).astype(np.float64)
            pi, hc0 = m['out16']
            hi, lo = (mainloop.f16(x.reshape(npix, -1)[:, hc0:hc0 + hid]).astype(np.float64) for x in planes[pi])
            rh = sig[:, hid:] * h
            # hi + lo holds the fp32 value to 2^-22 relative, and to 2^-25 absolute where lo is an fp16 subnormal
            tol = (0.25 * tb[:, hid:2 * hid] + ACT) * np.abs(h) + 2.0 ** -21 * np.abs(rh) + 2.0 ** -24
            against(hi + lo, rh, tol, slice(hid, 2 * hid), 'r * h')
            written16[pi][hc0:hc0 + hid] = True
        else:
            zb, hb, hid = m['gru']
            z = meta['bufs'][zb]['data'].reshape(npix, hid).astype(np.float64)
            h0 = meta['bufs'][hb]['data'].reshape(npix, hid).astype(np.float64)
            h = bufs[hb].reshape(npix, hid)
            want = (1 - z) * h0 + z * np.tanh(E[:, :hid])
            tol = z * (tb[:, :hid] + ACT) + 4 * U * (np.abs((1 - z) * h0) + np.abs(want))
            against(h, want, tol, slice(0, hid), 'hidden state')
            pi, hc0 = m['out16']
            eh, el = cases.split_f16(h)
            hi, lo = (x.reshape(npix, -1)[:, hc0:hc0 + hid] for x in planes[pi])
            assert np.array_equal(hi, eh.view(np.uint16)) and np.array_equal(lo, el.view(np.uint16)), where
            written16[pi][hc0:hc0 + hid] = True
    for i, P in enumerate(meta['planes']):
        if P['data'] is None:
            for x in planes[i]:
                assert (x[..., ~written16[i]] == mainloop.CANARY16).all(), f'{label}: fp16 canary overwritten (plane {i})'
    return worst


@pytest.mark.parametrize('case,kind', SWEEP, ids=[f"{c['name']}-{k}" for c, k in SWEEP])
def test_mainloop_sweep(runs, case, kind):
    c, meta, desc = runs[(case['name'], kind)]
    r = check_case(c, meta, desc, f"{case['name']}-{kind}")
    print(f"{case['name']}-{kind}: {desc[0]['total_chunks']} chunks, {desc[0]['nstages']} stages, group "
          f"{desc[0]['group_chunks']}, grid {desc[0]['grid']} of {desc[0]['items']} tiles: worst / bound {r:.4f}")


@pytest.mark.parametrize('case,kind', EPILOGUES, ids=[f"{c['name']}-{k}" for c, k in EPILOGUES])
def test_mainloop_epilogues(runs, case, kind):
    c, meta, desc = runs[(case['name'], kind)]
    r = check_case(c, meta, desc, f"{case['name']}-{kind}")
    print(f"{case['name']}-{kind}: worst / bound {r:.4f}")


@pytest.mark.parametrize('plan,kind', PLANS)
def test_mega_plans_equal_per_layer_kernels(runs, plan, kind):
    """The plan's per-layer run passes the model checks; every grid of the mega-kernel reproduces it bit for bit."""
    c, meta, desc = runs[(f'{plan}_conv', kind)]
    r = check_case(c, meta, desc, f'{plan}_conv-{kind}')
    ref = sorted(f for f in os.listdir(meta['dir']) if f.endswith('.bin') and f[0] in 'PB')
    for g in mainloop.MEGA_GRIDS:
        _, m2, d2 = runs[(f'{plan}_g{g}', kind)]
        for f in ref:
            a = np.fromfile(os.path.join(meta['dir'], f), np.uint8)
            b = np.fromfile(os.path.join(m2['dir'], f), np.uint8)
            assert np.array_equal(a, b), f'{plan} grid {d2[0]["grid"]}: {f} differs from the per-layer kernels'
    print(f'{plan}-{kind}: {len(desc)} layers, worst / bound {r:.4f}, grids {mainloop.MEGA_GRIDS} bit-identical')
