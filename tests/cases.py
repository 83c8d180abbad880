"""Seeded synthetic inputs shared by the golden generator and the parity tests.

Inputs are never stored: both sides regenerate them from the same NumPy PCG64 seeds
(SURVEY.md section 8(d)).  Only oracle OUTPUTS are committed under tests/golden/.
"""
import numpy as np

F32 = np.float32


def images(b, h, w, seed0=0, seed1=1):
    """README.md:99-100 style inputs: uniform [0, 255) float32 image pairs."""
    im1 = np.random.default_rng(seed0).uniform(0, 255, (b, h, w, 3)).astype(F32)
    im2 = np.random.default_rng(seed1).uniform(0, 255, (b, h, w, 3)).astype(F32)
    return im1, im2


def fmaps(b, h, w, c, seed=10):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((b, h, w, c)).astype(F32), rng.standard_normal((b, h, w, c)).astype(F32)


def lookup_coords(b, h, w, kind, seed=2):
    """Query coordinates for CorrBlock.retrieve.

    'grid'    : the integer pixel grid (iteration 0: every level-0 tap is exactly 0)
    'jitter'  : grid + U(-8, 8)^2 -- in and out of range, non-integer
    'edge'    : a mix that pins the quirks: exact integers, half-integers, exact borders, far outside
    """
    gy, gx = np.meshgrid(np.arange(h, dtype=F32), np.arange(w, dtype=F32), indexing='ij')
    grid = np.tile(np.stack([gx, gy], axis=-1)[None], (b, 1, 1, 1)).astype(F32)
    if kind == 'grid':
        return grid
    rng = np.random.default_rng(seed)
    if kind == 'jitter':
        return (grid + rng.uniform(-8, 8, grid.shape)).astype(F32)
    if kind == 'edge':
        c = (grid + rng.uniform(-3, 3, grid.shape)).astype(F32)
        flat = c.reshape(-1, 2)
        n = flat.shape[0]
        flat[0::7] = np.round(flat[0::7])                       # exact integers
        flat[1::7] = np.round(flat[1::7]) + F32(0.5)            # half integers (level-1 integers)
        flat[2::7, 0] = F32(w - 1)                              # right border
        flat[3::7, 1] = F32(0)                                  # top border
        flat[4::7] = flat[4::7] + F32(100)                      # far outside
        flat[5::7] = -flat[5::7] - F32(50)
        flat[6 % n::11] = np.round(flat[6 % n::11] * 4) / 4     # quarter integers (level-2 integers)
        return flat.reshape(c.shape)
    raise ValueError(kind)


def update_inputs(variant, b, h, w, seed=20):
    hid, ctx, cch = (128, 128, 324) if variant == 'raft' else (96, 64, 196)
    rng = np.random.default_rng(seed)
    net = np.tanh(rng.standard_normal((b, h, w, hid))).astype(F32)
    inp = np.maximum(rng.standard_normal((b, h, w, ctx)), 0).astype(F32)
    corr = (rng.standard_normal((b, h, w, cch)) * 3).astype(F32)
    flow = (rng.standard_normal((b, h, w, 2)) * 4).astype(F32)
    return net, inp, corr, flow


# ---------------------------------------------------------------------------------------------- geometry sweep
def tc_tile(h, w):
    """(TW, TH) pixel tile of every tensor-core convolution on an h x w grid: a Python mirror of tc_pick_tile
    (tf_raft_b200/csrc/conv_tc.cuh).  TW * TH = 128 with TW a power of two from 128 down to 8; the least padded area
    wins, and on a tie the wider tile (the first one tried)."""
    best = None
    tw = 128
    while tw >= 8:
        th = 128 // tw
        area = -(-w // tw) * tw * (-(-h // th) * th)
        if best is None or area < best[0]:
            best = (area, tw, th)
        tw //= 2
    return best[1], best[2]


# (B, h, w) update-block grids: one per tile shape, then one whose work list is many times the 132 SMs of an H100.  The
# 128 x 1 grid has 9 rows (not fewer) so that a 4-level pyramid, and with it the whole model loop, also runs on it.
TILE_GRIDS = (
    (2, 9, 128),       # 128 x 1 (the tile of the Sintel grid 56 x 128; TH = 1 gives the 5 x 1 GRU convolutions a 2-row halo)
    (2, 5, 40),        # 64 x 2
    (2, 9, 25),        # 32 x 4
    (3, 13, 11),       # 16 x 8
    (2, 9, 7),         # 8 x 16 (W <= 8, H >= 9)
    (4, 24, 40),       # 16 x 8, 36 pixel tiles per layer
)

# (B, h, w) lookup grids per pyramid depth.  Each has a deepest level of width or height 1; the second 4-level grid has
# every level width a multiple of 4 (the window kernel's 128-bit loads), the first has none.
LOOKUP_GRIDS = {
    1: ((2, 5, 7), (2, 1, 9)),
    2: ((2, 7, 3),),
    4: ((2, 9, 13), (1, 8, 32)),
    5: ((1, 17, 19),),
    6: ((1, 33, 37),),
}

# (B, h, w, C, levels) correlation pyramids: 1 to 6 levels (levels > 4 take the per-level pooling path of the tensor-core
# build), C from 64 to 256 (sqrt(C) a power of two or not), odd h and w, N = h*w never a multiple of 128.
PYRAMID_CASES = (
    (3, 9, 13, 64, 1),
    (3, 11, 7, 128, 2),
    (3, 15, 15, 192, 4),
    (3, 19, 23, 256, 4),
    (2, 31, 31, 256, 5),
    (1, 31, 95, 192, 5),
    (1, 63, 63, 64, 6),
    (1, 63, 63, 128, 6),
)


def level_sizes(h, w, levels):
    """(h, w) of every pyramid level: 2x2 VALID average pooling floors odd sizes (corr.py:113)."""
    return [(h >> l, w >> l) for l in range(levels)]


def lookup_path(B, h, w, levels, radius, out_stride, vec_ok=True):
    """The lookup kernel CorrBlock.retrieve and the loop launch for a B x h x w grid: a Python mirror of
    lookup_win_kernel (tf_raft_b200/csrc/lookup.cuh).  'window-vec' / 'window' = corr_lookup_win_kernel with 128-bit /
    scalar footprint loads, 'generic' = corr_lookup_kernel.  The window kernel exists for (radius, levels) = (4, 4) and
    (3, 4) and addresses the pyramid with 32-bit offsets, so it declines once level 0 (B*h*w planes of h*w elements) or
    the output (B*h*w rows of out_stride) holds 2^31 elements or more.  vec_ok: every level starts 16-byte aligned."""
    nq = B * h * w
    if levels != 4 or radius not in (3, 4) or nq * levels >= 2 ** 31:
        return 'generic'
    if nq * h * w >= 2 ** 31 or nq * out_stride >= 2 ** 31:
        return 'generic'
    vec = vec_ok and all(lw % 4 == 0 for _, lw in level_sizes(h, w, levels))
    return 'window-vec' if vec else 'window'


# (B, h, w) grids on both sides of the window kernel's 2^31-element limit on pyramid level 0, and one past 2^32: the
# pyramid (4 levels, fp32) takes 11.2 to 23.0 GB of device memory.
LARGE_CASES = (
    (1, 215, 215),     # images 1720 x 1720: B*N^2 = 2 136 750 625 < 2^31, window kernel, scalar loads
    (1, 216, 216),     # images 1728 x 1728: 2 176 782 336 >= 2^31, generic kernel
    (41, 56, 128),     # Sintel grid, batch 41: 2 106 589 184 < 2^31, window kernel, 128-bit loads
    (42, 56, 128),     # batch 42: 2 157 969 408 >= 2^31, generic kernel
    (1, 257, 256),     # 4 328 587 264 > 2^32, generic kernel
)


def boundary_queries(B, h, w):
    """Queries whose level-0 plane (elements [q*N, (q+1)*N) of the volume, N = h*w) holds element 2^31 or 2^32."""
    n = h * w
    return [e // n for e in (2 ** 31, 2 ** 32) if e < B * n * n]


def large_sample(B, h, w, n_random=32, seed=7):
    """Sorted query indices to check on a large grid: the first and last 4 queries of every image, each boundary query
    (boundary_queries) with its neighbours, and n_random seeded random queries."""
    n = h * w
    qs = set()
    for b in range(B):
        qs.update(range(b * n, b * n + 4))
        qs.update(range((b + 1) * n - 4, (b + 1) * n))
    for q in boundary_queries(B, h, w):
        qs.update(range(q - 1, q + 2))
    qs.update(np.random.default_rng(seed).integers(0, B * n, n_random).tolist())
    return np.array(sorted(q for q in qs if 0 <= q < B * n), dtype=np.int64)


def corr_rows(f1, f2, qs, levels):
    """float64 pyramid planes of the queries qs only: level 0 = f1[q] . f2[b]^T / sqrt(C) as an h x w plane, deeper
    levels pooled 2 x 2 VALID from it, the way oracle.raft_torch.CorrBlock pools.  f1, f2: (B, h, w, C) NumPy arrays.
    Returns levels tensors (len(qs), h_l, w_l, 1)."""
    import torch
    import torch.nn.functional as F
    B, h, w, c = f1.shape
    n = h * w
    qs = np.asarray(qs, dtype=np.int64)
    rows = torch.empty((len(qs), 1, h, w), dtype=torch.float64)
    for b in np.unique(qs // n):
        sel = np.nonzero(qs // n == b)[0]
        a = torch.from_numpy(f1[b].reshape(n, c)[qs[sel] - b * n]).double()
        t = torch.from_numpy(f2[b].reshape(n, c)).double()
        rows[torch.from_numpy(sel)] = ((a @ t.T) / np.sqrt(c)).reshape(len(sel), 1, h, w)
    out = [rows]
    for _ in range(levels - 1):
        out.append(F.avg_pool2d(out[-1], 2, 2))
    return [p.permute(0, 2, 3, 1) for p in out]


ENCODER_STAGES = {'raft': (64, ((64, 1), (96, 2), (128, 2))), 'small': (32, ((32, 1), (64, 2), (96, 2)))}


def encoder_plan(H, W, variant):
    """The tensor-core convolutions encoder_forward (tf_raft_b200/csrc/encoder.cuh) launches for an H x W image, in order:
    a Python mirror of its layer sequence and of enc_conv_tc's choices.  Each entry is a dict with the layer name, the
    kernel size k, the TMA element stride, the input (hin, win) and output (hout, wout) sizes, the pixel tile (tw, th)
    and the 'same' pads before (pt, pl).  The stem's 7 x 7 stride-2 window is gathered by stem_im2col_kernel into planes
    of the output's size, so the stem runs as a 1 x 1 stride-1 convolution; 1 x 1 convolutions are 'valid'.  Stride-2
    layers on an odd input pad one row / column on both sides, on an even input only after (TF 'same')."""
    c0, stages = ENCODER_STAGES[variant]
    h, w = -(-H // 2), -(-W // 2)
    plan = []

    def conv(name, k, stride, hin, win):
        hout, wout = -(-hin // stride), -(-win // stride)
        tw, th = tc_tile(hout, wout)
        # enc_conv_tc narrows a tile whose strided TMA box would pass 256 elements; tc_tile's widest tile is 128, so at
        # stride 2 the box is at most 256 wide and the rule never fires
        assert tw * stride <= 256 and th * stride <= 256
        if k == 1 or stride == 1:
            pt = pl = (k - 1) // 2
        else:
            pt = max((hout - 1) * stride + k - hin, 0) // 2
            pl = max((wout - 1) * stride + k - win, 0) // 2
        plan.append(dict(name=name, k=k, stride=stride, hin=hin, win=win, hout=hout, wout=wout, tw=tw, th=th,
                         pt=pt, pl=pl))
        return hout, wout

    conv('stem', 1, 1, h, w)
    for li, (c, s) in enumerate(stages, start=1):
        for bi, st in enumerate((s, 1)):
            p = f'layer{li}.{bi}'
            ho, wo = conv(p + '.conv1', 3, st, h, w)
            if st != 1:
                conv(p + '.downsample', 1, st, h, w)
            conv(p + '.conv2', 3, 1, ho, wo)
            h, w = ho, wo
    conv('conv2', 1, 1, h, w)
    return plan


def stride2_combos(H, W, variant, min_tiles=2):
    """(tw, th, odd input height, odd input width) of the stride-2 convolutions of encoder_plan(H, W, variant) whose
    output spans at least min_tiles pixel tiles in both directions."""
    return {(e['tw'], e['th'], e['hin'] % 2, e['win'] % 2) for e in encoder_plan(H, W, variant)
            if e['stride'] == 2 and -(-e['wout'] // e['tw']) >= min_tiles and -(-e['hout'] // e['th']) >= min_tiles}


# (H, W) images for the encoder geometry sweep (tests/test_gpu_encoders.py).  The first ten, a greedy cover found with
# encoder_plan over H in 8..400 and W in 8..1300, put a stride-2 layer on every (pixel tile, input-height parity,
# input-width parity) with the layer's output at least two tiles each way, for both encoders.  The last three are the
# smallest images: at 8 x 8 the last stage is 1 x 1, so instance norm sees one pixel and a zero variance.
ENCODER_GRIDS = (
    (17, 1283), (195, 129), (195, 135), (23, 1283), (97, 321), (49, 645), (99, 325), (103, 323), (35, 1029),
    (87, 1287),
    (8, 8), (8, 9), (9, 8),
)


def encoder_params(variant, norm_type, out_dim, seed=99, bias_scale=0.05, norm_jitter=0.2):
    """Parameters of a BasicEncoder ('raft') / SmallEncoder ('small') with any norm type, under the prefix 'enc.'."""
    from oracle import weights
    c0, stages = ENCODER_STAGES[variant]
    return weights.draw_params(weights.encoder_shapes('enc', norm_type, c0, stages, out_dim), seed, bias_scale, norm_jitter)


# ---------------------------------------------------------------------------------------------- value sweep
def split_f16(v):
    """NumPy emulation of the fp16 hi/lo operand split (split_f16, tf_raft_b200/csrc/common.cuh): values beyond fp16's
    range, +-inf included, saturate to +-65504, hi = fp16(v), lo = fp16(v - hi) with the difference taken in fp32.
    astype(np.float16) rounds to nearest even like __float2half_rn, subnormals included.  NaN stays NaN.  Returns
    (hi, lo) as float16 arrays."""
    v = np.asarray(v, dtype=F32)
    with np.errstate(invalid='ignore'):
        s = np.clip(v, F32(-65504), F32(65504)).astype(F32)
        hi = s.astype(np.float16)
        lo = (s - hi.astype(F32)).astype(np.float16)
    return hi, lo


def split_product(a, b):
    """float64 value of the three-pass product of a (M, K) and b (N, K) on split operands: hi.hi' + hi.lo' + lo.hi'
    (what the tensor-core kernels compute, up to their fp32 accumulation), and sum |a||b| over K, the scale of that
    accumulation's error.  Both (M, N)."""
    ah, al = (x.astype(np.float64) for x in split_f16(a))
    bh, bl = (x.astype(np.float64) for x in split_f16(b))
    return ah @ bh.T + ah @ bl.T + al @ bh.T, np.abs(a).astype(np.float64) @ np.abs(b).astype(np.float64).T


def dilate(mask, kh, kw, stride=1, padding='same'):
    """Receptive-field propagation through one convolution: mask (B, H, W) bool of the input pixels that hold a NaN ->
    the output pixels whose kh x kw window (Keras 'same' / 'valid' padding, stride 1 or 2, asymmetric 'same' padding
    for stride 2 as TF pads) reaches one.  Images never mix."""
    B, H, W = mask.shape
    if padding == 'same':
        ho, wo = -(-H // stride), -(-W // stride)
        pt = max((ho - 1) * stride + kh - H, 0) // 2
        pl = max((wo - 1) * stride + kw - W, 0) // 2
    else:
        ho, wo = (H - kh) // stride + 1, (W - kw) // stride + 1
        pt = pl = 0
    pad = np.zeros((B, pt + stride * ho + kh, pl + stride * wo + kw), dtype=bool)
    pad[:, pt:pt + H, pl:pl + W] = mask
    out = np.zeros((B, ho, wo), dtype=bool)
    for dy in range(kh):
        for dx in range(kw):
            out |= pad[:, dy:dy + stride * ho:stride, dx:dx + stride * wo:stride]
    return out


def encoder_field(mask):
    """dilate() through BasicEncoder / SmallEncoder without normalisation (extractor.py:113-130): the stem 7x7 s2, three
    stages of two residual blocks (3x3 convolutions, the first block of stages 2 and 3 with stride 2 and a 1x1 s2 VALID
    downsample on the skip path), then the 1x1 output convolution, which does not dilate."""
    m = dilate(mask, 7, 7, 2)
    for s in (1, 2, 2):
        for stride in (s, 1):
            fx = dilate(dilate(m, 3, 3, stride), 3, 3, 1)
            skip = dilate(m, 1, 1, stride, 'valid') if stride != 1 else m
            m = fx | skip
    return m


def update_field(variant, net, inp, corr, flow):
    """dilate() through the update block (update.py:70-153): per-pixel masks of the inputs -> masks of the new hidden
    state, of delta (the flow head's two 3x3 convolutions) and of the mask head (3x3, then 1x1).  1x1 convolutions
    (convc1 of both variants, mask.2) do not dilate."""
    if variant == 'raft':
        cor = dilate(dilate(corr, 1, 1, 1, 'valid'), 3, 3)
        flo = dilate(dilate(flow, 7, 7), 3, 3)
    else:
        cor = dilate(corr, 1, 1)
        flo = dilate(dilate(flow, 7, 7), 3, 3)
    x = dilate(cor | flo, 3, 3) | flow | inp
    passes = ((1, 5), (5, 1)) if variant == 'raft' else ((3, 3),)
    h = net
    for kh, kw in passes:
        zr = dilate(h | x, kh, kw)
        q = dilate(zr | h | x, kh, kw)
        h = h | zr | q
    return h, dilate(dilate(h, 3, 3), 3, 3), dilate(h, 3, 3)
