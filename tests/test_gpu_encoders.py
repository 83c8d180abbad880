"""The tensor-core encoders (tf_raft_b200/csrc/encoder.cuh) against the oracle run in float64.

Under the default precision ('f16x2') RAFT and SmallRAFT run fnet and cnet on these encoders, and bench.py times them:
fnet on 2B images, cnet on B.  The tests below compare them with `oracle.raft_torch.encoder` in torch.float64 on the
GPU (TF32 does not apply to float64), at

- every stride-2 pixel tile and edge parity the host can pick (cases.ENCODER_GRIDS, checked by
  tests/test_geometry_cases.py), with every norm, raw and normalised input, biases and jittered norm parameters;
- the production shapes: the benchmark's batches at 448 x 512 and 448 x 1024, KITTI and 1080p sizes, and training-mode
  BatchNorm whose one statistics group spans a whole batch of 448 x 1024 images;
- hard normalisation statistics: channel means far from zero, dead channels, and a flat map with one bright corner;
- every output width the ABI accepts.

Tiles never straddle images and statistics are per image, so an image's output must not depend on the rest of the batch,
bit for bit.  Each comparison also prints the fp32 oracle's error against the same truth (cuDNN in IEEE fp32), which shows
how much of the tolerance an fp32 computation needs by itself.
"""
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import cases
import probe_build
from oracle import raft_torch as rt

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
F32, F64 = np.float32, torch.float64
TOL = 2e-4                     # the encoder tolerance of tests/test_gpu_stages.py and tests/test_gpu_geometry.py
OUT_DIM = {('raft', 'fnet'): 256, ('raft', 'cnet'): 256, ('small', 'fnet'): 128, ('small', 'cnet'): 160}
NORMS = {'instance': ('instance', False), 'batch-inference': ('batch', False), 'batch-training': ('batch', True),
         'none': (None, False)}


@pytest.fixture(scope='module')
def T():
    import tf_raft_b200
    from tf_raft_b200 import _lib
    from tf_raft_b200.layers.extractor import force_ieee_fp32
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    force_ieee_fp32()
    return tf_raft_b200


def _id(g):
    return 'x'.join(map(str, g))


def maxabs(a, b):
    return float((a.double() - b.double()).abs().max())


def normalised(im):
    """2 * (x / 255) - 1 in float32, the arithmetic of the encoders' raw-image load (model.py:70-71)."""
    return 2 * (torch.from_numpy(im) / 255.0) - 1.0


def oracle(p, x, norm, training, dtype):
    """oracle.raft_torch.encoder on the GPU: p holds CUDA tensors, x is an NHWC float32 tensor -> NHWC output."""
    x = x.cuda().permute(0, 3, 1, 2).to(dtype)
    return rt.encoder(rt.Ops(p, dtype), x, 'enc', norm, training).permute(0, 2, 3, 1)


def encoder(variant, norm, out_dim, p):
    from tf_raft_b200.layers.extractor import BasicEncoder, SmallEncoder
    enc = (BasicEncoder if variant == 'raft' else SmallEncoder)(output_dim=out_dim, norm_type=norm, backend='native')
    enc.load_params(p, 'enc.')
    return enc


def cuda_params(p):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in p.items()}


def check(tag, got, x, p, norm, training, gate=None):
    """got against the fp64 oracle of the normalised input x; prints the error next to the fp32 oracle's.  gate: a
    function of (fp64 truth, fp32 oracle error) -> tolerance; TOL by default."""
    pc = cuda_params(p)
    truth = oracle(pc, x, norm, training, F64)
    e32 = maxabs(oracle(pc, x, norm, training, torch.float32), truth)
    assert tuple(got.shape) == tuple(truth.shape)
    e = maxabs(got, truth)
    tol = TOL if gate is None else gate(truth, e32)
    print(f'[{tag}] max-abs {e:.2e} (fp32 oracle {e32:.2e}, tolerance {tol:.1e}), '
          f'|out| up to {float(truth.abs().max()):.2f}')
    assert e <= tol, (tag, e, tol)
    return truth


def test_gpu_fp64_oracle_equals_the_cpu_one(T):
    """The fp64 truth run on the GPU (cuDNN / CUDA float64) is the CPU one to 1e-10, on an odd size with every norm."""
    for norm, (nt, training) in NORMS.items():
        p = cases.encoder_params('small', nt, 64, seed=3)
        im, _ = cases.images(2, 37, 45, seed0=11)
        x = normalised(im)
        cpu = rt.encoder(rt.Ops(p, F64), x.permute(0, 3, 1, 2).double(), 'enc', nt, training).permute(0, 2, 3, 1)
        gpu = oracle(cuda_params(p), x, nt, training, F64).cpu()
        e = maxabs(gpu, cpu)
        print(f'[fp64 gpu vs cpu] norm {norm}: max-abs {e:.1e}')
        assert e <= 1e-10


# --------------------------------------------------------------------------------------------- 1. geometry sweep
@pytest.mark.parametrize('size', cases.ENCODER_GRIDS, ids=_id)
@pytest.mark.parametrize('norm', list(NORMS))
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_encoder_geometry_sweep(T, variant, norm, size):
    """Every stride-2 pixel tile on even and odd input heights and widths, each spanning two or more tiles both ways, and
    the 8 x 8, 8 x 9 and 9 x 8 images (a 1 x 1 last stage).  Batch 2 of distinct images, biases, jittered gamma, beta and
    moving statistics; the image raw (0..255) and normalised."""
    H, W = size
    nt, training = NORMS[norm]
    out_dim = OUT_DIM[(variant, 'fnet')]
    p = cases.encoder_params(variant, nt, out_dim, seed=7 * H + W)
    im, _ = cases.images(2, H, W, seed0=H * W)
    assert not np.array_equal(im[0], im[1])
    x = normalised(im)
    enc = encoder(variant, nt, out_dim, p)
    got = {raw: enc(torch.from_numpy(im if raw else x.numpy()).cuda(), training=training, raw_image=raw)
           for raw in (True, False)}
    truth = check(f'sweep {variant} {norm} {H}x{W} raw', got[True], x, p, nt, training)
    e = maxabs(got[False], truth)
    print(f'[sweep {variant} {norm} {H}x{W} normalised] max-abs {e:.2e}')
    assert e <= TOL


# --------------------------------------------------------------------------------------------- 2. production shapes
PRODUCTION = (
    ('raft', 'fnet', 8, 448, 512), ('raft', 'cnet', 4, 448, 512),          # bench.py: batch 4 at 448 x 512
    ('raft', 'fnet', 4, 448, 1024), ('raft', 'cnet', 2, 448, 1024),        # Sintel, padded
    ('small', 'fnet', 8, 448, 512), ('small', 'cnet', 4, 448, 512),
    ('raft', 'fnet', 2, 376, 1248), ('raft', 'cnet', 2, 376, 1248),        # KITTI, padded
    ('raft', 'fnet', 1, 1088, 1920), ('raft', 'cnet', 1, 1088, 1920),      # 1080p, padded
)


@pytest.mark.parametrize('variant,which,n,H,W', PRODUCTION, ids=['-'.join(map(str, c)) for c in PRODUCTION])
def test_encoder_production_shapes(T, variant, which, n, H, W):
    """The encoders as the models call them (the model's norm, raw images, inference) at the batches and sizes users
    run: at fnet 8 x 448 x 512 the stem alone is 3584 tiles of 128 x 1, some 27 per persistent CTA on 132 SMs."""
    nt = rt.VARIANTS[variant]['fnorm' if which == 'fnet' else 'cnorm']
    out_dim = OUT_DIM[(variant, which)]
    p = cases.encoder_params(variant, nt, out_dim, seed=H + n)
    im, _ = cases.images(n, H, W, seed0=W + n)
    got = encoder(variant, nt, out_dim, p)(torch.from_numpy(im).cuda(), training=False, raw_image=True)
    check(f'production {variant}.{which} ({nt}) {n}x{H}x{W}', got, normalised(im), p, nt, False)


def test_encoder_training_batchnorm_over_a_large_batch(T):
    """cnet with training-mode BatchNorm at 8 x 448 x 1024: one statistics group of 8 x 224 x 512 = 917 504 pixels per
    channel after the stem."""
    n, H, W = 8, 448, 1024
    p = cases.encoder_params('raft', 'batch', 256, seed=5)
    im, _ = cases.images(n, H, W, seed0=12)
    got = encoder('raft', 'batch', 256, p)(torch.from_numpy(im).cuda(), training=True, raw_image=True)
    check(f'production raft.cnet (batch, training) {n}x{H}x{W}', got, normalised(im), p, 'batch', True)


# --------------------------------------------------------------------------------------------- 3. bit-exact invariants
@pytest.mark.parametrize('norm', ['instance', 'batch-inference', 'none'])
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_encoder_images_are_independent_of_the_batch(T, variant, norm):
    """Without batch statistics an image's output is a function of that image alone: image b of a batch of 8 equals the
    image run by itself, a reversed batch gives the reversed outputs, and two runs are identical, all bit for bit."""
    nt, training = NORMS[norm]
    out_dim = OUT_DIM[(variant, 'fnet')]
    H, W = 99, 325                                                     # several tiles both ways at every layer
    p = cases.encoder_params(variant, nt, out_dim, seed=17)
    im, _ = cases.images(8, H, W, seed0=23)
    enc = encoder(variant, nt, out_dim, p)

    def run(a):
        return enc(torch.from_numpy(np.ascontiguousarray(a)).cuda(), training=training, raw_image=True).cpu()
    full = run(im)
    assert torch.equal(run(im), full), 'two runs differ'
    assert torch.equal(run(im[::-1]), full.flip(0)), 'a reversed batch does not give the reversed outputs'
    for b in range(8):
        assert torch.equal(run(im[b:b + 1]), full[b:b + 1]), f'image {b} alone differs from image {b} of the batch'


# --------------------------------------------------------------------------------------------- 4. statistics edges
def stats_gate(truth, e32):
    """Where fp32 itself loses digits (a mean of 1e3 against a spread of 1), the kernel may lose what the fp32 oracle
    loses, four times over."""
    return max(TOL * max(1.0, float(truth.abs().max())), 4 * e32)


@pytest.mark.parametrize('norm', ['instance', 'batch-training'])
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_encoder_statistics_far_from_zero(T, variant, norm):
    """Stem biases of +-1e3 and stem weights a tenth of their usual size: every channel's mean is 1e3 away from zero,
    some thousand times its standard deviation."""
    nt, training = NORMS[norm]
    out_dim = OUT_DIM[(variant, 'fnet')]
    p = cases.encoder_params(variant, nt, out_dim, seed=31)
    c0 = p['enc.conv1.bias'].shape[0]
    p['enc.conv1.bias'] = np.where(np.arange(c0) % 2, 1e3, -1e3).astype(F32)
    p['enc.conv1.kernel'] = (p['enc.conv1.kernel'] * 0.1).astype(F32)
    H, W = 195, 135
    im, _ = cases.images(2, H, W, seed0=37)
    got = encoder(variant, nt, out_dim, p)(torch.from_numpy(im).cuda(), training=training, raw_image=True)
    check(f'stats far means {variant} {norm}', got, normalised(im), p, nt, training, stats_gate)


@pytest.mark.parametrize('norm', ['instance', 'batch-training'])
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_encoder_statistics_of_dead_channels(T, variant, norm):
    """Output channels whose kernel is all zero (every 7th of the stem, every 5th of stage 2's first convolution) hold
    their bias everywhere: zero variance, so the norm's output there is beta, which needs the mean exact."""
    nt, training = NORMS[norm]
    out_dim = OUT_DIM[(variant, 'fnet')]
    p = cases.encoder_params(variant, nt, out_dim, seed=41)
    for name, step in (('enc.conv1.kernel', 7), ('enc.layer2.0.conv1.kernel', 5)):
        k = p[name].copy()
        k[..., ::step] = 0
        p[name] = k
    H, W = 97, 321
    im, _ = cases.images(2, H, W, seed0=43)
    got = encoder(variant, nt, out_dim, p)(torch.from_numpy(im).cuda(), training=training, raw_image=True)
    check(f'stats dead channels {variant} {norm}', got, normalised(im), p, nt, training, stats_gate)


@pytest.mark.parametrize('size', [(448, 512), (1088, 1920)], ids=_id)
def test_encoder_instance_norm_of_a_bright_corner(T, size):
    """A flat image (0 plus noise of 1e-3, normalised input, so the zero padding matches the background) with 2 x 2 unit
    pixels in its top-left corner, in image 1 of 2 only.  The stem's first output pixel, where every statistics thread of
    the first split starts, is then hundreds of standard deviations from its channel's mean.  Image 0 also checks that
    the images' statistics stay apart.  The normalised corner dominates the output (|out| up to some 250), so a
    tolerance relative to the output's magnitude would pass statistics a hundred times worse than fp32's; the native
    encoder must stay within TOL or eight times the fp32 oracle's error."""
    H, W = size
    p = cases.encoder_params('raft', 'instance', 256, seed=47)
    x = (np.random.default_rng(H).standard_normal((2, H, W, 3)) * 1e-3).astype(F32)
    x[1, :2, :2, :] = 1.0
    got = encoder('raft', 'instance', 256, p)(torch.from_numpy(x).cuda(), training=False, raw_image=False)
    check(f'stats bright corner {H}x{W}', got, torch.from_numpy(x), p, 'instance', False,
          lambda truth, e32: max(TOL, 8 * e32))


# --------------------------------------------------------------------------------------------- 5. output widths
@pytest.mark.parametrize('out_dim', range(32, 257, 32))
@pytest.mark.parametrize('variant', ['raft', 'small'])
def test_encoder_output_widths(T, variant, out_dim):
    """Every out_dim raft_b200_encoder_forward accepts (32 to 256 in steps of 32): partial 32-column epilogue chunks
    (224 is a 112-column tile) and widths the models never use."""
    H, W = 195, 135
    p = cases.encoder_params(variant, 'instance', out_dim, seed=out_dim)
    im, _ = cases.images(2, H, W, seed0=53)
    got = encoder(variant, 'instance', out_dim, p)(torch.from_numpy(im).cuda(), training=False, raw_image=True)
    check(f'width {variant} {out_dim}', got, normalised(im), p, 'instance', False)


# --------------------------------------------------------------------------------------------- 6. the statistics kernels
@pytest.fixture(scope='module')
def stats_probe():
    exe = probe_build.build(os.path.join(ROOT, 'tests', 'norm_stats_probe.cu'), 'raft_norm_stats_probe')
    assert exe is not None, 'nvcc not found'
    return exe


def stats_data(kind, P, C, seed):
    """(1, P, C) float32 raw convolution output of one image: N(0, 1) noise; noise + 1e3; or a flat map (sigma 0.01)
    with 16 pixels raised by 50, at pixel 0 (the first sample of the first split's statistics threads) or inside the
    sixth split."""
    y = np.random.default_rng(seed).standard_normal((1, P, C))
    if kind == 'offset':
        y += 1e3
    elif kind.startswith('spike'):
        y *= 1e-2
        at = 0 if kind == 'spike-first' else (P // 64) * 5 + 17
        y[:, at:at + 16] += 50.0
    return y.astype(F32)


STATS_CASES = [(kind, P, 64) for P in (224 * 256, 544 * 960) for kind in ('noise', 'offset', 'spike-first', 'spike-mid')]
STATS_CASES += [(kind, 224 * 256, C) for C in (96, 256) for kind in ('noise', 'spike-first')]


@pytest.mark.parametrize('kind,P,C', STATS_CASES, ids=['-'.join(map(str, c)) for c in STATS_CASES])
def test_norm_statistics_against_fp64(stats_probe, kind, P, C):
    """norm_stats_kernel + norm_final_kernel on the stem outputs of 448 x 512 (P = 224 x 256) and 1088 x 1920
    (544 x 960) images: per-channel mean and variance against float64 on the same float32 data.  A sum shifted by a
    sample far from the mean (a bright pixel where a thread starts) cancels: 3e-4 relative error on the variance at
    1088 x 1920 before the running-mean shift, where torch's fp32 variance stays near 3e-8."""
    y = stats_data(kind, P, C, seed=P + C)
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, 'y.bin'), os.path.join(d, 'out.bin')
        y.tofile(src)
        res = subprocess.run([stats_probe, src, dst, '1', str(P), str(C)], capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stderr
        out = np.fromfile(dst, dtype=F32)
    mean, var = out[:C].astype(np.float64), out[C:].astype(np.float64) ** -2
    y64 = y[0].astype(np.float64)
    m64, v64 = y64.mean(axis=0), y64.var(axis=0)
    y32 = torch.from_numpy(y[0])
    v32 = y32.var(dim=0, unbiased=False).double().numpy()
    e_var, e32 = float(np.max(np.abs(var - v64) / v64)), float(np.max(np.abs(v32 - v64) / v64))
    e_mean = np.abs(mean - m64)
    print(f'[statistics {kind} P={P} C={C}] variance relative error {e_var:.2e} (torch fp32 {e32:.2e}), '
          f'mean error / std {float(np.max(e_mean / np.sqrt(v64))):.2e}')
    assert e_var <= 2e-6
    assert np.all(e_mean <= 1e-6 * np.sqrt(v64) + 2.0 ** -22 * np.abs(m64))
