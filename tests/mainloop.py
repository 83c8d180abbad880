"""Cases, case files and the fp64 model of the shared wgmma mainloop (tests/conv_tc_probe.cu), used by
tests/test_gpu_mainloop.py (on the GPU) and tests/test_mainloop_cases.py (coverage and model, on the CPU).

A case is one probe run: operand planes, fp32 buffers and one or more layers, each a conv_tc_kernel launch (mode 'conv')
or an item range of one update_mega_kernel launch (mode 'mega').  `sweep()` is the covering design of the mainloop's
configuration space; `model()` computes, from the exact fp16 operands the MMAs read, per output in fp64

    E = 2^-k * sum(a_hi w_hi + a_hi w_lo + a_lo w_hi) + bias      S = 2^-k * sum(|a_hi w_hi| + |a_hi w_lo| + |a_lo w_hi|) + |bias|

as im2col GEMMs: every product of two fp16 values is exact in fp64, so E is the split arithmetic itself, not the fp32
truth.
"""
import os

import numpy as np

import cases

F32 = np.float32
U = 2.0 ** -24
SMS = 132                                          # H100 SXM: the grid `0` (one CTA per SM) in the coverage checks
CANARY16 = 0x7e5a
CANARY32 = 0x7fc0cafe
EPI_LINEAR, EPI_GRU_ZR, EPI_GRU_Q = 0, 1, 2
# Ring depth tc_finalize derives for a column tile of bn (conv_tc.cuh: stages of 2 * 16 KiB + 256 * bn bytes in
# 227 KiB less 33.5 KiB of staging, alignment slack and barriers, at most 8).
MAX_STAGES = {bn: min(8, (227 * 1024 - 34304) // (32768 + 256 * bn)) for bn in range(16, 129, 16)}


def mma_n(bn):
    return next(n for n in (16, 32, 64, 96, 128) if bn <= n)


def out_hw(h, w, stride):
    return -(-h // stride), -(-w // stride)


def same_pads(k, hin, hout, stride):
    """Keras 'same' pad before, the way enc_conv_tc computes it (stride 1: (k - 1) / 2)."""
    if stride == 1:
        return (k - 1) // 2
    return max((hout - 1) * stride + k - hin, 0) // 2


# ------------------------------------------------------------------------------------------------------------ specs
def conv(name, taps, stride, segs, bn, ntn, n_total, img, group, nstages=0, grid=0, seg_c0=None, nw=1, cinmap=None,
         flatten=False, f32=(0, 0), h_c0=0):
    """One conv_tc_kernel layer.  segs: 64-channel chunks per tap of each K segment (one plane each); seg_c0: first
    channel each segment reads (its plane is that much wider); img: (B, Hin, Win); f32: (extra row stride, c0) of the
    fp32 output; h_c0: first channel of the hi/lo output plane; cinmap: (n0, n1, dst1) two-range TcCinMap of n0 + n1
    source channels; flatten: taps over 2 channels flattened into the channel axis (a 1 x 1 layer on im2col planes)."""
    return dict(name=name, mode='conv', grid=grid, layers=[dict(
        taps=taps, stride=stride, segs=tuple(segs), seg_c0=tuple(seg_c0 or (0,) * len(segs)), bn=bn, ntn=ntn,
        n_total=n_total, img=img, group=group, nstages=nstages, nw=nw, cinmap=cinmap, flatten=flatten, f32=f32,
        h_c0=h_c0, epi='plain', src=None, deps=())])


def sweep():
    """The covering design: each MMA width at every ring depth, each (taps, stride, K segments) form, every relation of
    chunks per tile to ring depth and to promotion group, every grid with more tiles than CTAs, every pixel tile on a
    ragged image.  test_mainloop_cases.py checks the coverage from the probe's own geometry."""
    S = []
    # (MMA width, ring depth) pairs; tap shapes, strides and segments rotate through them
    S += [conv('w16_s2', (1, 1), 1, (1,), 16, 2, 20, (2, 33, 45), 1, 2, 1),
          conv('w16_s3', (1, 1), 1, (3,), 16, 1, 9, (2, 7, 41), 2, 3, 2, f32=(3, 1)),
          conv('w16_s4', (1, 1), 1, (5,), 16, 3, 40, (1, 19, 23), 4, 4, 3, seg_c0=(64,)),
          conv('w16_s5', (1, 5), 1, (2,), 16, 1, 11, (1, 9, 70), 10, 5, 7, f32=(8, 8)),
          conv('w16_s5_sms', (1, 1), 1, (1,), 16, 1, 13, (1, 137, 128), 2, 5, 0),
          conv('w32_s2', (3, 3), 1, (2,), 32, 1, 27, (2, 11, 29), 19, 2, 1, h_c0=32),
          conv('w32_s3', (3, 3), 2, (1,), 32, 2, 50, (1, 33, 45), 5, 3, 3),
          conv('w32_s4', (5, 1), 1, (1,), 32, 3, 70, (1, 18, 21), 3, 4, 2, h_c0=8),
          conv('w48_s2', (1, 1), 2, (1,), 48, 3, 130, (2, 16, 30), 1, 2, 2, f32=(5, 3)),
          conv('w48_s3', (7, 7), 2, (1,), 48, 1, 37, (1, 27, 40), 5, 3, 1),
          conv('w48_s4', (1, 1), 1, (4,), 48, 2, 90, (3, 5, 66), 3, 4, 7, nw=2),
          conv('w64_s2', (1, 5), 1, (1, 2), 64, 1, 61, (1, 14, 50), 2, 2, 3, seg_c0=(0, 64)),
          conv('w64_s3', (3, 3), 1, (1, 3), 64, 2, 100, (1, 21, 19), 35, 3, 2, seg_c0=(64, 0)),
          conv('w64_s4', (3, 3), 1, (3, 1), 64, 1, 50, (1, 10, 33), 36, 4, 1, cinmap=(150, 30, 192), nw=2),
          conv('w80_s2', (5, 1), 1, (1, 1), 80, 1, 77, (2, 9, 17), 11, 2, 1, h_c0=32),
          conv('w80_s3', (1, 1), 2, (1, 1), 80, 2, 150, (1, 25, 27), 1, 3, 3, seg_c0=(0, 128)),
          conv('w96_s2', (3, 3), 2, (1,), 96, 1, 90, (2, 24, 34), 2, 2, 7),
          conv('w96_s3', (1, 1), 1, (3, 1), 96, 1, 95, (1, 5, 130), 5, 3, 2),
          conv('w112_s2', (1, 1), 1, (3,), 112, 2, 200, (1, 31, 9), 2, 2, 1),
          conv('w112_s3', (1, 5), 2, (1,), 112, 1, 100, (1, 10, 63), 5, 3, 2),
          conv('w128_s2', (1, 1), 1, (3,), 128, 3, 300, (1, 6, 67), 1, 2, 3),
          conv('w128_s3', (7, 7), 1, (1,), 128, 1, 120, (1, 12, 12), 5, 3, 1)]
    # the remaining (taps, stride, segments) forms, the flattened im2col layer and the default ring depth
    S += [conv('t3x3_s2_seg2', (3, 3), 2, (1, 1), 64, 1, 40, (1, 17, 31), 2, 0, 2, seg_c0=(64, 0)),
          conv('t1x5_s2_seg2', (1, 5), 2, (2, 1), 32, 2, 60, (1, 16, 24), 3, 0, 3),
          conv('t5x1_s2', (5, 1), 2, (2,), 48, 1, 44, (2, 19, 10), 5, 0, 1),
          conv('t5x1_s2_seg2', (5, 1), 2, (1, 1), 16, 1, 15, (1, 30, 31), 2, 0, 7),
          conv('t7x7_s1_seg2', (7, 7), 1, (1, 1), 32, 1, 30, (1, 9, 20), 5, 0, 2),
          conv('t7x7_s2_seg2', (7, 7), 2, (1, 1), 16, 1, 12, (1, 20, 17), 3, 0, 1),
          conv('flatten7x7', (7, 7), 1, (2,), 64, 2, 120, (1, 13, 14), 2, 0, 3, flatten=True)]
    return S


def epilogue_cases():
    """Each epilogue at two widths: EPI_LINEAR with every option, the GRU gates, and the fused advance."""
    def lin(name, bn, ntn, n_total, res_stride, res_c0):
        c = conv(name, (3, 3), 1, (2,), bn, ntn, n_total, (1, 10, 27), 2, f32=(4, 0))
        c['layers'][0].update(epi='linear', res=(res_stride, res_c0))
        return c

    def gru(name, mode, bn, ntn, hid):
        c = conv(name, (1, 5), 1, (1, 1), bn, ntn, 2 * hid if mode == EPI_GRU_ZR else hid, (1, 9, 30), 2)
        c['layers'][0].update(epi=('zr', 'q')[mode - 1], hid=hid)
        return c

    def adv(name, bn):
        c = conv(name, (3, 3), 1, (1,), bn, 1, 2, (2, 7, 19), 2)
        c['layers'][0].update(epi='advance')
        return c
    return [lin('epi_linear_64', 64, 2, 100, 107, 3), lin('epi_linear_32', 32, 1, 30, 40, 8),
            gru('epi_zr_64', EPI_GRU_ZR, 64, 1, 32), gru('epi_zr_96', EPI_GRU_ZR, 96, 2, 96),
            gru('epi_q_32', EPI_GRU_Q, 32, 2, 64), gru('epi_q_96', EPI_GRU_Q, 96, 1, 96),
            adv('epi_advance_16', 16), adv('epi_advance_32', 32)]


def mega_plans():
    """Synthetic update_mega_kernel plans.  'carve': a 3 x 3 layer, a two-source nseg = 2 layer reading its output, a
    5 x 1 layer, a 1 x 1 bn = 16 layer of one-chunk items: stage sizes 48, 64, 40 and 36 KiB, so the ring is re-carved at
    every layer change.  'deep': one-chunk items at the deepest ring, so the producer runs as far ahead as it can."""
    def L(taps, segs, seg_c0, src, bn, ntn, n_total, out, nstages=0, deps=()):
        return dict(taps=taps, stride=1, segs=segs, seg_c0=seg_c0, bn=bn, ntn=ntn, n_total=n_total, img=(2, 40, 64),
                    group=2, nstages=nstages, nw=1, cinmap=None, flatten=False, f32=(0, 0), h_c0=0, epi='plain',
                    src=src, out=out, deps=deps)
    carve = [L((3, 3), (1,), (64,), ('in',), 64, 1, 60, 'p1'),
             L((3, 3), (1, 1), (0, 0), ('p1', 'in'), 128, 1, 128, 'p2', deps=((0, 0, 0),)),
             L((5, 1), (2,), (0,), ('p2',), 32, 2, 50, 'p3', deps=((1, 0, 0),)),
             L((1, 1), (1,), (0,), ('p3',), 16, 1, 13, 'f32', deps=((2, 0, 0),))]
    deep = [L((1, 1), (1,), (0,), ('in',), 16, 3, 40, 'f32', nstages=5),
            L((1, 1), (1,), (0,), ('in',), 16, 1, 9, 'f32', nstages=5),
            L((1, 1), (1,), (0,), ('in',), 16, 2, 30, 'f32', nstages=5)]
    return {'carve': carve, 'deep': deep}


MEGA_GRIDS = (1, 2, 3, 7, 0)


def mega_case(name, plan, mode, grid):
    return dict(name=name, mode=mode, grid=grid, layers=[dict(l) for l in plan])


# ------------------------------------------------------------------------------------------------------- case files
def _geometry(l):
    B, hin, win = l['img']
    ho, wo = out_hw(hin, win, l['stride'])
    kh, kw = (1, 1) if l['flatten'] else l['taps']
    return B, hin, win, ho, wo, kh, kw, same_pads(kh, hin, ho, l['stride']), same_pads(kw, win, wo, l['stride'])


def _weights_dims(l):
    """(list of (kh, kw, cin, cout) of the packed sources, cin_pad, cout_pad, TcCinMap line or None)."""
    cin_pad = 64 * sum(l['segs'])
    kh, kw = l['taps']
    if l['flatten']:
        cin = 2
        assert kh * kw * cin <= cin_pad
    elif l['cinmap']:
        n0, n1, d1 = l['cinmap']
        cin = n0 + n1
        assert n0 <= d1 and d1 + n1 <= cin_pad
    else:
        cin = cin_pad
    cout = l['n_total']
    couts = [cout] if l['nw'] == 1 else [cout // 2, cout - cout // 2]
    cmap = None
    if l['cinmap']:
        n0, n1, d1 = l['cinmap']
        cmap = (2, 0, n0, 0, n0, n1, d1)
    return [(kh, kw, cin, c) for c in couts], cin_pad, l['ntn'] * l['bn'], cmap


def build(case, kind, seed, root=None):
    """case.txt text for `case` and, with root, the case directory with seeded operands of data kind 'a' (small
    integers), 'b' (positive) or 'c' (N(0, 1)).  Returns (text, meta): meta names every plane and buffer and holds the
    fp32 inputs the checks need."""
    rng = np.random.default_rng(seed)
    lines = [f"mode {case['mode']}", f"grid {case['grid']}"]
    planes, bufs = [], []
    meta = dict(kind=kind, layers=[], planes=planes, bufs=bufs)
    d = None
    if root is not None:
        d = os.path.join(root, case['name'] + '_' + kind)
        os.makedirs(d, exist_ok=True)

    def save(arr, fname):
        if d is not None:
            np.ascontiguousarray(arr, dtype=F32).tofile(os.path.join(d, fname))

    def act(shape):
        if kind == 'a':
            return rng.integers(-8, 9, shape).astype(F32)
        if kind == 'b':
            return rng.uniform(0.25, 2.0, shape).astype(F32)
        return rng.standard_normal(shape).astype(F32)

    def plane(B, H, W, C, cs, data):
        i = len(planes)
        fname = '-' if data is None else f'act{i}.bin'
        if data is not None:
            save(data, fname)
        planes.append(dict(B=B, H=H, W=W, C=C, cs=cs, data=data))
        lines.append(f'plane {B} {H} {W} {C} {cs} {fname}')
        return i

    def buf(n, data=None):
        i = len(bufs)
        fname = '-' if data is None else f'buf{i}.bin'
        if data is not None:
            save(data, fname)
        bufs.append(dict(n=n, data=data))
        lines.append(f'buf {n} {fname}')
        return i

    named = {}
    for li, l in enumerate(case['layers']):
        B, hin, win, ho, wo, kh, kw, ph, pw = _geometry(l)
        npix = B * ho * wo
        m = dict(spec=l, npix=npix, geometry=(B, hin, win, ho, wo, kh, kw, ph, pw))
        # operand planes
        segp = []
        for s, (ch, c0) in enumerate(zip(l['segs'], l['seg_c0'])):
            src = l['src'][s] if l['src'] else None
            if src in named:
                segp.append(named[src])
                continue
            cs = c0 + 64 * ch
            segp.append(plane(B, hin, win, cs, cs, act((B, hin, win, cs))))
            if src:
                named[src] = segp[-1]
        m['seg_planes'] = segp
        # weights
        dims, cin_pad, cout_pad, cmap = _weights_dims(l)
        ws, bs = [], []
        lay = [f'layer']
        for j, (wkh, wkw, cin, cout) in enumerate(dims):
            shape = (wkh, wkw, cin, cout)
            if kind == 'a':
                w = rng.integers(-7, 8, shape).astype(F32)
                w.flat[rng.integers(0, w.size)] = 7.0 * (1 - 2 * (j % 2))   # max |w| = 7 in every layer
                b = np.zeros(cout, F32)
            elif kind == 'b':
                # outputs of order 1 whatever K, so that layers fed by other layers stay inside fp16's range
                w = (rng.uniform(0.25, 1.0, shape) / (wkh * wkw * cin)).astype(F32)
                b = rng.uniform(0.0, 1.0, cout).astype(F32)
            else:
                w = (rng.standard_normal(shape) / np.sqrt(cin * wkh * wkw)).astype(F32)
                b = (rng.standard_normal(cout) * 0.1).astype(F32)
            if l['epi'] in ('zr', 'q'):                      # gates of order 1: the fast activations see their range
                w = (w / np.float32(max(1.0, np.abs(w).sum(axis=(0, 1, 2)).max() / 4))).astype(F32)
            ws.append(w)
            bs.append(b)
            save(w, f'L{li}_w{j}.bin')
            save(b, f'L{li}_b{j}.bin')
            lay.append(f'wsrc {wkh} {wkw} {cin} {cout} L{li}_w{j}.bin L{li}_b{j}.bin')
        m.update(w=ws, b=bs, cin_pad=cin_pad, cout_pad=cout_pad, cmap=cmap)
        lay.append(f"pack {cin_pad} {cout_pad} {int(l['flatten'])}")
        if cmap:
            lay.append('cinmap ' + ' '.join(map(str, cmap)))
        for s, ch in enumerate(l['segs']):
            lay.append(f"seg {segp[s]} {l['seg_c0'][s]} {ch}")
        lay.append(f"geom {B} {ho} {wo} {l['stride']} {ph} {pw} 0 0")
        lay.append(f"tile {l['bn']} {l['ntn']} {l['n_total']}")
        lay.append(f"group {l['group']}")
        if l['nstages']:
            lay.append(f"nstages {l['nstages']}")
        for dep in l['deps']:
            lay.append('dep ' + ' '.join(map(str, dep)))
        # epilogue and outputs
        epi, n_total = l['epi'], l['n_total']
        out = l.get('out', 'both')
        if epi in ('plain', 'linear'):
            mode, act_, oscale = EPI_LINEAR, int(epi == 'linear'), (0.25 if epi == 'linear' else 1.0)
        elif epi == 'zr':
            mode, act_, oscale = EPI_GRU_ZR, 0, 1.0
        elif epi == 'q':
            mode, act_, oscale = EPI_GRU_Q, 0, 1.0
        else:
            mode, act_, oscale = EPI_LINEAR, 0, 1.0
        lay.append(f'epi {mode} {act_} {oscale}')
        m.update(mode=mode, act=act_, out_scale=oscale)
        ext = 7                                              # fp32 rows past the last pixel: must stay canaries
        if mode == EPI_LINEAR and out in ('both', 'f32'):
            f32_stride = n_total + l['f32'][0] + l['f32'][1]
            m['out32'] = (buf((npix + ext) * f32_stride), f32_stride, l['f32'][1])
            lay.append(f"out32 {m['out32'][0]} {f32_stride} {l['f32'][1]}")
        if out in ('both', 'p1', 'p2', 'p3') and epi != 'advance':
            width = l['hid'] if mode != EPI_LINEAR else cout_pad
            cs = -(-(l['h_c0'] + width) // 64) * 64
            pi = plane(B, ho, wo, cs, cs, None)
            if out != 'both':
                named[out] = pi
            m['out16'] = (pi, l['h_c0'])
            lay.append(f"out16 {pi} {l['h_c0']}")
        if epi == 'linear':
            sc = rng.uniform(0.5, 1.5, cout_pad + 64).astype(F32)
            sh = rng.uniform(-0.5, 0.5, cout_pad + 64).astype(F32)
            rs, rc0 = l['res']
            res = rng.standard_normal(((npix + ext) * rs,)).astype(F32)
            cat = rng.standard_normal((npix * 2,)).astype(F32)
            m['post'] = (buf(sc.size, sc), buf(sh.size, sh))
            m['residual'] = (buf(res.size, res), rs, rc0)
            m['concat'] = (buf(cat.size, cat), 2)
            lay += [f"post {m['post'][0]} {m['post'][1]}", f"residual {m['residual'][0]} {rs} {rc0}",
                    f"concat {m['concat'][0]} 2"]
        if epi in ('zr', 'q'):
            hid = l['hid']
            z = rng.uniform(0, 1, (npix * hid,)).astype(F32)
            h = np.tanh(rng.standard_normal((npix * hid,))).astype(F32)
            m['gru'] = (buf(z.size, z if mode == EPI_GRU_Q else None), buf(h.size, h), hid)
            lay.append(f"gru {m['gru'][0]} {m['gru'][1]} {hid}")
        if epi == 'advance':
            c1 = (rng.uniform(-5, 40, (npix * 2,))).astype(F32)
            m['adv'] = (buf(c1.size, c1), buf(npix * 2))
            lay.append(f"adv {m['adv'][0]} {m['adv'][1]}")
        lines += lay
        meta['layers'].append(m)
    text = '\n'.join(lines) + '\n'
    if d is not None:
        with open(os.path.join(d, 'case.txt'), 'w') as f:
            f.write(text)
    meta['dir'] = d
    return text, meta


# ------------------------------------------------------------------------------------------------------------- model
def f16(bits):
    return np.asarray(bits, dtype=np.uint16).view(np.float16)


def im2col(plane, seg_c0, chunks, kh, kw, ph, pw, stride, ho, wo):
    """(taps, B * ho * wo, K) operand of every tap: the TMA box of the tap, zero outside the image, with the segments'
    channels concatenated.  plane: list of (B, H, W, cs) arrays, one per segment."""
    out = []
    for ty in range(kh):
        for tx in range(kw):
            cols = []
            for p, c0, ch in zip(plane, seg_c0, chunks):
                B, H, W, _ = p.shape
                pad = np.zeros((B, H + kh + stride * ho, W + kw + stride * wo, 64 * ch), p.dtype)
                pad[:, ph:ph + H, pw:pw + W] = p[..., c0:c0 + 64 * ch]
                cols.append(pad[:, ty:ty + stride * ho:stride, tx:tx + stride * wo:stride].reshape(B * ho * wo, -1))
            out.append(np.concatenate(cols, axis=1))
    return out


def model(a_hi, a_lo, seg_c0, chunks, geometry, w_hi, w_lo, inv_scale, bias):
    """E and S (npix, cout_pad) in float64 from the fp16 operands (a_*: one (B, H, W, cs) float16 array per segment;
    w_*: (taps, cout_pad, cin_pad) float16) and the fp32 bias (cout_pad)."""
    B, hin, win, ho, wo, kh, kw, ph, pw, stride = geometry
    d = lambda x: [np.asarray(v, np.float64) for v in x]
    ah = im2col(d(a_hi), seg_c0, chunks, kh, kw, ph, pw, stride, ho, wo)
    al = im2col(d(a_lo), seg_c0, chunks, kh, kw, ph, pw, stride, ho, wo)
    wh, wl = np.asarray(w_hi, np.float64), np.asarray(w_lo, np.float64)
    E = np.zeros((B * ho * wo, wh.shape[1]))
    S = np.zeros_like(E)
    for t in range(kh * kw):
        E += ah[t] @ wh[t].T + ah[t] @ wl[t].T + al[t] @ wh[t].T
        S += np.abs(ah[t]) @ np.abs(wh[t]).T + np.abs(ah[t]) @ np.abs(wl[t]).T + np.abs(al[t]) @ np.abs(wh[t]).T
    b = np.asarray(bias, np.float64)
    return E * inv_scale + b, S * inv_scale + np.abs(b)


def bound(S, total, group):
    """|got - E| <= 2u (12 g + n_groups + 2) S: see test_gpu_mainloop.py."""
    g = min(group, total)
    return 2 * U * (12 * g + -(-total // group) + 2) * S


def packed_expected(ws, cin_pad, cout_pad, cmap, flatten):
    """The [tap][cout_pad][cin_pad] hi / lo planes tc_pack_weights writes for the HWIO sources ws (concatenated along
    cout), 2^k (max |w| 2^k in [2^12, 2^13)) and the unscaled fp32 planes."""
    m = max(float(np.abs(w).max()) for w in ws)
    k = 0
    if m > 0:
        k = max(-24, min(24, 13 - int(np.frexp(m)[1])))
    s = F32(2.0 ** k)
    kh, kw = (1, 1) if flatten else ws[0].shape[:2]
    full = np.zeros((kh * kw, cout_pad, cin_pad), F32)
    off = 0
    for w in ws:
        wkh, wkw, cin, cout = w.shape
        w2 = w.reshape(kh * kw, -1, cout)                   # flatten: (1, kh * kw * cin, cout)
        if cmap:
            _, s0, n0, d0, s1, n1, d1 = cmap
            for src0, n, dst0 in ((s0, n0, d0), (s1, n1, d1)):
                full[:, off:off + cout, dst0:dst0 + n] = np.transpose(w2[:, src0:src0 + n], (0, 2, 1))
        else:
            full[:, off:off + cout, :w2.shape[1]] = np.transpose(w2, (0, 2, 1))
        off += cout
    hi, lo = cases.split_f16(full * s)
    return hi, lo, float(s), full


def total_chunks(l):
    kh, kw = (1, 1) if l['flatten'] else l['taps']
    return kh * kw * sum(l['segs'])
