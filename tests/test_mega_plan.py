"""update_mega_kernel's work list is race-free: every pair of conflicting items is ordered by its waits (CPU).

update_mega_kernel (tf_raft_b200/csrc/mega.cuh) runs every tensor-core layer of one update-block application in one
launch; CTAs claim (layer, column tile, pixel tile) items in list order, and the only order between two items is the
completion counters an item's producer waits on before its loads.  A missing wait shows on the GPU only when the timing
happens to expose it, so the suite's output comparisons cannot be relied on to see one.  The plan, though, is pure host
code: tests/mega_plan_probe.cu builds it through update_core_tc exactly as the library does (fake device addresses,
nothing launched) and prints it, and this module checks it exactly.

The checker restates in Python what each item reads and writes and which counters it waits on and publishes.  That
restatement follows the device code:
  * waits: the producer loop of update_mega_kernel (mega.cuh:110-129), counters indexed with the CONSUMER's tile grid;
    publishing: the consumer warps' red.release after the epilogue (mega.cuh:165-171); items decoded by tc_decode_tile
    (conv_tc.cuh:461-469) and located by mega_layer_of (mega.cuh:54-58);
  * reads: the TMA boxes of tc_produce_tile (conv_tc.cuh:373-392): for every segment, whole 64-channel chunks
    [seg_c0, seg_c0 + 64 * chunks) over the tile widened by the taps (ph before, kh - 1 - ph after; pw likewise), clipped
    to the image (TMA zero-fills outside it);
  * epilogue, per 32-column chunk of every pixel of the tile inside the image (tc_consume_tile, conv_tc.cuh:409-444, and
    tc_epilogue_regs, conv_tc.cuh:118-286):
      EPI_LINEAR  concat columns past n_total read concat_src (W.flow); fp32 output only up to n_total; fp16 planes in
                  whole 32-column chunks (zero and concat columns past n_total included); the fused advance, on column 0
                  only, reads and writes coords1 and writes W.flow;
      EPI_GRU_ZR  columns below hid write z; the others read fp32 h and write r*h to the output plane;
      EPI_GRU_Q   read z and h, write h in place and its output plane.
A change to the wait loop, the publishing code, the TMA boxes or the epilogue's loads and stores is therefore NOT
covered by this test: it must update this restatement in the same change (the GPU tests still exercise the device code
itself).  Host-side changes -- the rows of kBasicTc / kSmallTc (update.cuh), mega_add (mega.cuh), the workspace layout
and the tile choice -- are covered, because the plan is dumped from the library's own host code.

Checks per case: (a) every waited-on counter lies in its source layer's range and exactly one item of that layer
publishes it, so no wait can be left pending; (b) every wait names a lower item number; (c) every conflicting pair of
items (same buffer, overlapping pixels and channels, at least one write) is ordered by the transitive closure of the
waits; (d) nflags + 1 <= W.mega_flag_words; (e) every (layer, column tile, pixel tile) item appears once and each layer's
writes cover its output columns over the whole grid.  Also checked: every operand map and output pointer addresses the
plane or buffer that the row names, with the stride the kernel assumes.
"""
import functools
import json
import os
import subprocess

import numpy as np
import pytest

import cases
import probe_build

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
PROBE_SRC = os.path.join(ROOT, 'tests', 'mega_plan_probe.cu')

EPI_LINEAR, EPI_GRU_ZR, EPI_GRU_Q = 0, 1, 2
TC_CONCAT_FLOW, TC_ADVANCE, TC_MASK_ONLY, TC_MASK_TAIL = 1, 2, 4, 8
PLANES = ('corr', 'cor1', 'cf', 'flo1', 'x', 'h16', 'rh', 'fm', 'fim')     # TcPlane order (update.cuh)
OUT_DELTA, OUT_MASK = 9, 10
CONSUMER_WARPS = 8

# (B, h, w): one grid per tile shape (TH = 1 gives the 5 x 1 GRU convolutions a 2-tile halo), the benchmark grid, the
# Sintel grid, an odd grid and a single pixel; then, for every tile width, a grid of several tile columns: only there do
# the 1 x 5 convolutions' horizontal halos reach a neighbouring tile.
GRIDS = tuple(dict.fromkeys(tuple(cases.TILE_GRIDS) + ((4, 56, 64), (1, 56, 128), (3, 13, 11), (1, 1, 1)) +
                            ((1, 9, 256), (1, 9, 192), (1, 8, 96), (1, 32, 24))))
FORMS = (('basic', 1), ('basic', 0), ('small', 0))          # (variant, mask head)
CASES = [(v, b, h, w, m, a) for (b, h, w) in GRIDS for (v, m) in FORMS for a in (1, 0)]


# ---------------------------------------------------------------------------------------------------------------- probe
@pytest.fixture(scope='module')
def probe():
    exe = probe_build.build(PROBE_SRC, 'raft_mega_plan_probe')
    if exe is None:
        pytest.skip('nvcc not found: the plan probe cannot be built')
    return exe


@functools.lru_cache(maxsize=None)
def _dump_text(exe, variant, B, h, w, mask, adv):
    res = subprocess.run([exe, variant, str(B), str(h), str(w), str(mask), str(adv)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return res.stdout


def dump(exe, variant, B, h, w, mask, adv):
    """The plan as a fresh dict (callers may corrupt their copy)."""
    return json.loads(_dump_text(exe, variant, B, h, w, mask, adv))


# ------------------------------------------------------------------------------------------------------------- checker
class Buffers:
    """Address -> buffer name, and every buffer's channel stride.  fp16 planes: hi address (lo checked alongside)."""

    def __init__(self, plan):
        self.plane_of = {}
        self.stride = {}
        self.lo = {}
        for k, (hi, lo, s) in enumerate(plan['planes']):
            if hi:
                self.plane_of[hi] = PLANES[k]
                self.lo[PLANES[k]] = lo
            self.stride[PLANES[k]] = s
        hid = plan['hid']
        f32 = plan['f32']
        self.f32_of = {f32[n]: n for n in ('h', 'z', 'flow', 'coords1', 'delta', 'mask')}
        self.stride.update(h=hid, z=hid, flow=2, coords1=2, delta=2, mask=576)


def layer_accesses(plan, L, bufs, problems):
    """The footprint of one item of layer L as a function of its tile: returns f(nt, b, ty, tx) -> list of
    (buffer, write, b, y0, y1, x0, x1, c0, c1), half-open ranges.  Pointer / map mismatches go to `problems`."""
    lay = plan['layers'][L]
    tab = lay['table']
    H, W, TH, TW = lay['H'], lay['W'], lay['TH'], lay['TW']
    bn, n_total, mode = lay['bn'], lay['n_total'], lay['mode']
    name = 'layer %d' % L

    def bad(msg):
        problems.append('%s: %s' % (name, msg))

    if lay['stride'] != 1:
        bad('stride %d (the update blocks run stride 1)' % lay['stride'])
    # operand segments: the tensor map must address the row's plane, with the plane's stride, hi/lo pair and tile box
    segs = []
    for s in range(lay['nseg']):
        m = lay['a_map'][s]
        plane = bufs.plane_of.get(m['addr'])
        if plane is None:
            bad('segment %d map addresses no operand plane' % s)
            continue
        if s < len(tab['segs']) and PLANES[tab['segs'][s][0]] != plane:
            bad('segment %d reads %s, the row names %s' % (s, plane, PLANES[tab['segs'][s][0]]))
        if m['dims'] != [bufs.stride[plane], W, H, lay['B'], 2] or m['box'] != [64, TW, TH, 1, 2] or \
                m['strides'][3] != bufs.lo[plane] - m['addr']:
            bad('segment %d map of %s: dims %s box %s' % (s, plane, m['dims'], m['box']))
        c0, c1 = lay['seg_c0'][s], lay['seg_c0'][s] + 64 * lay['seg_chunks'][s]
        if c1 > bufs.stride[plane]:
            bad('segment %d reads channels [%d, %d) of %s (stride %d)' % (s, c0, c1, plane, bufs.stride[plane]))
        segs.append((plane, c0, c1))
    if len(segs) != len(tab['segs']) or any(list(t[1:]) != [c0, (c1 - c0) // 64]
                                            for t, (_, c0, c1) in zip(tab['segs'], segs)):
        bad('segments %s differ from the row %s' % (segs, tab['segs']))

    def f32(addr, what):
        n = bufs.f32_of.get(addr)
        if n is None:
            bad('%s points at no fp32 buffer' % what)
        return n

    out_plane = bufs.plane_of.get(lay['out_hi']) if lay['out_hi'] else None
    if lay['out_hi'] and (out_plane is None or bufs.lo[out_plane] != lay['out_lo'] or
                          lay['h_stride'] != bufs.stride[out_plane]):
        bad('fp16 output does not address an operand plane with its stride')
        out_plane = None
    if tab['out'] < len(PLANES) and out_plane != PLANES[tab['out']]:
        bad('writes plane %s, the row names %s' % (out_plane, PLANES[tab['out']]))
    out_f32 = f32(lay['out_f32'], 'out_f32') if lay['out_f32'] else None
    if out_f32 is not None and lay['f32_stride'] != bufs.stride[out_f32]:
        bad('fp32 output stride %d, %s has %d' % (lay['f32_stride'], out_f32, bufs.stride[out_f32]))
    if tab['out'] == OUT_DELTA and out_f32 != 'delta' or tab['out'] == OUT_MASK and out_f32 != 'mask':
        bad('fp32 output is %s' % out_f32)
    if lay['residual']:
        bad('a residual input is not part of the update-block epilogues this checker restates')
    concat = f32(lay['concat_src'], 'concat_src') if lay['concat_src'] else None
    if bool(tab['flags'] & TC_CONCAT_FLOW) != (concat == 'flow'):
        bad('concat source %s' % concat)
    adv = None
    if lay['adv_coords']:
        adv = (f32(lay['adv_coords'], 'adv_coords'), f32(lay['adv_flow'], 'adv_flow'))
        if adv != ('coords1', 'flow') or not (tab['flags'] & TC_ADVANCE) or n_total != 2 or mode != EPI_LINEAR:
            bad('fused advance on %s' % (adv,))
    if mode != EPI_LINEAR:
        zb, hb = f32(lay['z'], 'z'), f32(lay['h'], 'h')
        if (zb, hb) != ('z', 'h') or lay['hid'] != plan['hid'] or out_plane is None:
            bad('GRU epilogue operands z=%s h=%s hid=%d' % (zb, hb, lay['hid']))
    # the 32-column chunks one thread handles: (column offset in the tile, ncol)
    chunks = [(c0, min(32, bn - c0)) for cb in range(0, bn, 64) for c0 in (cb, cb + 32) if c0 < bn]
    ph, pw, kh, kw = lay['ph'], lay['pw'], lay['kh'], lay['kw']
    hid = plan['hid']

    def accesses(nt, b, ty, tx):
        acc = []
        # TMA boxes: rows y0 - ph .. y0 + TH - 1 + (kh - 1 - ph), clipped (out-of-image is zero fill, not a read)
        ry0, ry1 = max(0, ty * TH - ph), min(H, ty * TH + TH + kh - 1 - ph)
        rx0, rx1 = max(0, tx * TW - pw), min(W, tx * TW + TW + kw - 1 - pw)
        for plane, c0, c1 in segs:
            acc.append((plane, False, b, ry0, ry1, rx0, rx1, c0, c1))
        y0, y1, x0, x1 = ty * TH, min(H, ty * TH + TH), tx * TW, min(W, tx * TW + TW)
        if y0 >= y1 or x0 >= x1:
            return acc
        t = (b, y0, y1, x0, x1)
        for c0, ncol in chunks:
            col = nt * bn + c0
            if mode == EPI_LINEAR:
                if concat and col + 32 > n_total:
                    a0, a1 = max(0, col - n_total), min(lay['concat_n'], col + 32 - n_total)
                    if a0 < a1:
                        acc.append((concat, False) + t + (a0, a1))
                nvalid = min(ncol, n_total - col)
                if out_f32 and nvalid > 0:
                    acc.append((out_f32, True) + t + (lay['f32_c0'] + col, lay['f32_c0'] + col + nvalid))
                if out_plane and ncol == 32:
                    acc.append((out_plane, True) + t + (lay['h_c0'] + col, lay['h_c0'] + col + 32))
                if adv and col == 0:
                    acc.append(('coords1', False) + t + (0, 2))
                    acc.append(('coords1', True) + t + (0, 2))
                    acc.append(('flow', True) + t + (0, 2))
            elif mode == EPI_GRU_ZR:
                if col < hid:
                    acc.append(('z', True) + t + (col, col + 32))
                else:
                    hc = col - hid
                    acc.append(('h', False) + t + (hc, hc + 32))
                    acc.append((out_plane, True) + t + (lay['h_c0'] + hc, lay['h_c0'] + hc + 32))
            else:
                acc.append(('z', False) + t + (col, col + 32))
                acc.append(('h', False) + t + (col, col + 32))
                acc.append(('h', True) + t + (col, col + 32))
                acc.append((out_plane, True) + t + (lay['h_c0'] + col, lay['h_c0'] + col + 32))
        return acc

    return accesses


def decode(lay, t):
    """tc_decode_tile (conv_tc.cuh:461-469)."""
    mtiles = lay['B'] * lay['tiles_y'] * lay['tiles_x']
    nt, mt = divmod(t, mtiles)
    mt, tx = divmod(mt, lay['tiles_x'])
    b, ty = divmod(mt, lay['tiles_y'])
    return nt, b, ty, tx


def layer_of(plan, item):
    """mega_layer_of (mega.cuh:54-58)."""
    L = 0
    layers = plan['layers']
    while L + 1 < len(layers) and item >= layers[L + 1]['item0']:
        L += 1
    return L


def items_of(plan):
    return [(i, layer_of(plan, i)) + decode(plan['layers'][layer_of(plan, i)], i - plan['layers'][layer_of(plan, i)]['item0'])
            for i in range(plan['nitems'])]


def published_flag(lay, nt, b, ty, tx):
    """The counter an item's consumer warps increment (mega.cuh:165-171)."""
    mtiles = lay['B'] * lay['tiles_y'] * lay['tiles_x']
    return lay['flag0'] + nt * mtiles + (b * lay['tiles_y'] + ty) * lay['tiles_x'] + tx


def waited_flags(plan, lay, nt, b, ty, tx):
    """(source layer, counter) of every wait of one item: the producer loop of mega.cuh:110-129, which indexes the
    source's counters with the consumer's own tile grid."""
    out = []
    mtiles = lay['B'] * lay['tiles_y'] * lay['tiles_x']
    for d in range(lay['ndep']):
        src = lay['dep_layer'][d]
        SL = plan['layers'][src]
        for n in range(lay['dep_nlo'][d], lay['dep_nhi'][d] + 1):
            for yy in range(max(0, ty - lay['dep_ry']), min(lay['tiles_y'] - 1, ty + lay['dep_ry']) + 1):
                for xx in range(max(0, tx - lay['dep_rx']), min(lay['tiles_x'] - 1, tx + lay['dep_rx']) + 1):
                    out.append((src, SL['flag0'] + n * mtiles + (b * lay['tiles_y'] + yy) * lay['tiles_x'] + xx))
    return out


def _overlap(a, b):
    return a[2] == b[2] and a[3] < b[4] and b[3] < a[4] and a[5] < b[6] and b[5] < a[6] and a[7] < b[8] and b[7] < a[8]


def check(plan, drop=()):
    """Problems found in the plan (empty: race-free) and the figures of the case.  drop: (waiting item, publishing item)
    wait edges to leave out, for the checker's own tests."""
    problems = []
    layers = plan['layers']
    bufs = Buffers(plan)
    items = items_of(plan)
    acc_fn = [layer_accesses(plan, L, bufs, problems) for L in range(len(layers))]

    # (e) the work list: layers back to back, every (layer, nt, tile) once
    pos = 0
    for L, lay in enumerate(layers):
        if lay['item0'] != pos:
            problems.append('layer %d starts at item %d, the list is at %d' % (L, lay['item0'], pos))
        pos = lay['item0'] + lay['B'] * lay['tiles_y'] * lay['tiles_x'] * lay['n_tiles_n']
        if (lay['B'], lay['H'], lay['W'], lay['TH'], lay['TW']) != (plan['B'], plan['h'], plan['w'], layers[0]['TH'],
                                                                    layers[0]['TW']):
            problems.append('layer %d runs another tile grid' % L)
    if pos != plan['nitems']:
        problems.append('the layers hold %d items, nitems = %d' % (pos, plan['nitems']))
    seen = {}
    for i, L, nt, b, ty, tx in items:
        key = (L, nt, b, ty, tx)
        if key in seen or not (0 <= nt < layers[L]['n_tiles_n']):
            problems.append('item %d repeats or lies outside %s' % (i, key))
        seen[key] = i
    for L, lay in enumerate(layers):
        want = lay['B'] * lay['tiles_y'] * lay['tiles_x'] * lay['n_tiles_n']
        got = sum(1 for k in seen if k[0] == L)
        if got != want:
            problems.append('layer %d has %d items, not %d' % (L, got, want))

    # (a) / (d) counters: every item publishes its own, inside [0, nflags) (flags[nflags] is the claim cursor)
    publisher = {}
    for i, L, nt, b, ty, tx in items:
        f = published_flag(layers[L], nt, b, ty, tx)
        publisher.setdefault(f, []).append(i)
        if not 0 <= f < plan['nflags']:
            problems.append('item %d publishes counter %d outside [0, nflags = %d)' % (i, f, plan['nflags']))
    if plan['nflags'] + 1 > plan['mega_flag_words']:
        problems.append('nflags + 1 = %d > mega_flag_words = %d' % (plan['nflags'] + 1, plan['mega_flag_words']))

    # waits -> edges; (a) each resolves to exactly one publisher of the source layer, (b) which comes earlier
    preds = [set() for _ in items]
    drop = set(drop)
    for i, L, nt, b, ty, tx in items:
        for src, f in waited_flags(plan, layers[L], nt, b, ty, tx):
            SL = layers[src]
            n_src = SL['B'] * SL['tiles_y'] * SL['tiles_x'] * SL['n_tiles_n']
            pubs = publisher.get(f, [])
            if not SL['flag0'] <= f < SL['flag0'] + n_src:
                problems.append('item %d waits on counter %d outside layer %d\'s range' % (i, f, src))
            if len(pubs) != 1 or items[pubs[0]][1] != src:
                problems.append('item %d waits on counter %d, published by items %s, not by one item of layer %d'
                                % (i, f, pubs, src))
                continue
            p = pubs[0]
            if p >= i:
                problems.append('item %d waits on item %d, not an earlier one' % (i, p))
                continue
            if (i, p) not in drop:
                preds[i].add(p)

    # transitive closure: ancestor bitsets in list order (every edge points to a lower item)
    anc = [0] * len(items)
    for i in range(len(items)):
        a = 0
        for p in preds[i]:
            a |= anc[p] | (1 << p)
        anc[i] = a

    # footprints, bucketed by (buffer, image, pixel tile) so that only neighbours are compared
    TH, TW = layers[0]['TH'], layers[0]['TW']
    buckets = {}
    footprint = []
    for i, L, nt, b, ty, tx in items:
        fp = acc_fn[L](nt, b, ty, tx)
        footprint.append(fp)
        for a in fp:
            if a[8] > bufs.stride[a[0]] or a[7] < 0:
                problems.append('item %d: channels [%d, %d) of %s (stride %d)' % (i, a[7], a[8], a[0], bufs.stride[a[0]]))
            for cy in range(a[3] // TH, (a[4] - 1) // TH + 1):
                for cx in range(a[5] // TW, (a[6] - 1) // TW + 1):
                    buckets.setdefault((a[0], a[2], cy, cx), []).append((i, a))

    # (c) conflicts: same buffer, overlapping pixels and channels, at least one write -> ordered by the waits
    conflicts = set()
    for entries in buckets.values():
        for k, (i, a) in enumerate(entries):
            for j, c in entries[k + 1:]:
                if i != j and (a[1] or c[1]) and _overlap(a, c):
                    conflicts.add((min(i, j), max(i, j), a[0]))
    pairs = {(i, j) for i, j, _ in conflicts}
    for i, j, buf in sorted(conflicts):
        if not (anc[j] >> i) & 1:
            Li, Lj = items[i][1], items[j][1]
            problems.append('items %d (layer %d, nt/b/ty/tx %s) and %d (layer %d, %s) conflict on %s with no wait '
                            'between them' % (i, Li, items[i][2:], j, Lj, items[j][2:], buf))

    # (e) every layer's writes cover its output columns over the whole grid
    for L, lay in enumerate(layers):
        tab = lay['table']
        n_out = tab['n_total'] - (tab['bn'] if (tab['flags'] & TC_MASK_TAIL) and not plan['mask'] else 0)
        if lay['n_total'] != n_out:
            problems.append('layer %d: n_total %d, the row promises %d columns' % (L, lay['n_total'], n_out))
        want = {}
        if lay['mode'] == EPI_LINEAR:
            if lay['out_hi'] and bufs.plane_of.get(lay['out_hi']):
                cat = lay['concat_n'] if lay['concat_src'] else 0
                want[bufs.plane_of[lay['out_hi']]] = (lay['h_c0'], lay['h_c0'] + n_out + cat)
            if lay['out_f32'] and bufs.f32_of.get(lay['out_f32']):
                want[bufs.f32_of[lay['out_f32']]] = (lay['f32_c0'], lay['f32_c0'] + n_out)
            if lay['adv_coords']:
                want['coords1'] = want['flow'] = (0, 2)
        else:
            hid = plan['hid']
            plane = PLANES[tab['out']]
            want = {'z': (0, hid), plane: (lay['h_c0'], lay['h_c0'] + hid)} if lay['mode'] == EPI_GRU_ZR else \
                {'h': (0, hid), plane: (lay['h_c0'], lay['h_c0'] + hid)}
        if not want:
            problems.append('layer %d writes nothing' % L)
        cover = {buf: np.zeros((plan['B'], plan['h'], plan['w'], c1 - c0), bool) for buf, (c0, c1) in want.items()}
        for i in range(lay['item0'], lay['item0'] + lay['B'] * lay['tiles_y'] * lay['tiles_x'] * lay['n_tiles_n']):
            for buf, wr, b, y0, y1, x0, x1, c0, c1 in footprint[i] if i < len(footprint) else ():
                if wr and buf in cover:
                    w0, w1 = want[buf]
                    if max(c0, w0) < min(c1, w1):
                        cover[buf][b, y0:y1, x0:x1, max(c0, w0) - w0:min(c1, w1) - w0] = True
        for buf, m in cover.items():
            if not m.all():
                problems.append('layer %d leaves %d of %d output elements of %s unwritten'
                                % (L, int((~m).sum()), m.size, buf))

    edges = sum(len(p) for p in preds)
    unneeded = sum(1 for i, p in enumerate(preds) for q in p if (q, i) not in pairs)
    return problems, dict(items=len(items), edges=edges, conflicts=len(pairs), waits_without_conflict=unneeded)


# ---------------------------------------------------------------------------------------------------------------- tests
def _id(c):
    v, b, h, w, m, a = c
    return '%s%s-%dx%dx%d-%s' % (v, '+mask' if m else '', b, h, w, 'advance' if a else 'noadvance')


@pytest.mark.parametrize('case', CASES, ids=[_id(c) for c in CASES])
def test_mega_plan_is_race_free(probe, case):
    plan = dump(probe, *case)
    problems, stats = check(plan)
    print('%s: %d items, %d wait edges, %d conflicting pairs checked, %d waits between items that do not conflict '
          'directly' % (_id(case), stats['items'], stats['edges'], stats['conflicts'], stats['waits_without_conflict']))
    assert not problems, '\n'.join(problems[:20]) + ('\n... %d problems' % len(problems) if len(problems) > 20 else '')
    assert stats['conflicts'] > 0 or plan['nitems'] == 0


def _layer(plan, kw, kh, mode):
    """Index of the (only) planned layer with this kernel shape and epilogue."""
    (L,) = [i for i, l in enumerate(plan['layers']) if (l['kw'], l['kh'], l['mode']) == (kw, kh, mode)]
    return L


def test_checker_reports_a_dropped_edge(probe):
    plan = dump(probe, 'basic', 2, 5, 40, 1, 1)
    assert not check(plan)[0]
    zr2 = _layer(plan, 1, 5, EPI_GRU_ZR)           # z|r2 (5 x 1) reads PL_H where q1 (1 x 5) wrote it, tile for tile
    q1 = _layer(plan, 5, 1, EPI_GRU_Q)
    i, p = plan['layers'][zr2]['item0'], plan['layers'][q1]['item0']
    problems, _ = check(plan, drop=[(i, p)])
    assert any('items %d ' % p in m and 'and %d ' % i in m for m in problems), problems


def test_checker_reports_a_lowered_row_halo_at_th1(probe):
    plan = dump(probe, 'basic', *cases.TILE_GRIDS[0], 1, 1)
    assert plan['layers'][0]['TH'] == 1 and not check(plan)[0]
    zr2 = _layer(plan, 1, 5, EPI_GRU_ZR)
    assert plan['layers'][zr2]['dep_ry'] == 2
    plan['layers'][zr2]['dep_ry'] = 1
    problems, _ = check(plan)
    assert any('conflict on h16' in m for m in problems), problems


def test_checker_reports_a_shifted_flag0(probe):
    plan = dump(probe, 'small', 3, 13, 11, 0, 1)
    assert not check(plan)[0]
    for L in range(len(plan['layers'])):
        bad = json.loads(json.dumps(plan))
        bad['layers'][L]['flag0'] += 1
        problems, _ = check(bad)
        assert any('published by items' in m or 'outside [0, nflags' in m for m in problems), (L, problems)


def test_checker_reports_a_narrowed_mask2_range(probe):
    plan = dump(probe, 'basic', 4, 24, 40, 1, 0)
    assert not check(plan)[0]
    mask2 = len(plan['layers']) - 1
    assert plan['layers'][mask2]['table']['flags'] & TC_MASK_ONLY
    lay = plan['layers'][mask2]
    assert (lay['dep_nlo'][0], lay['dep_nhi'][0]) == (2, 3)
    lay['dep_nhi'][0] = 2                           # columns [256, 384) of fh1|m0, not [256, 512)
    problems, _ = check(plan)
    assert any('conflict on fm' in m for m in problems), problems
