"""CPU: the NumPy restatement of torchvision's ColorJitter on PIL images (oracle/pil_colour_np.py), which the GPU kernels
are held to, against Pillow and torchvision themselves: Image.blend over every pair of bytes, RGB->L, RGB->HSV and
HSV->RGB over every input, hue shifts, the contrast mean on a tie, and the whole jitter in all 24 op orders; then the
colour='torchvision' sampler's draws against ColorJitter.get_params and the original RAFT's augmentors
(oracle/raft_augment.py)."""
import itertools

import numpy as np
import pytest
import torch

from oracle import pil_colour_np as P

Image = pytest.importorskip('PIL.Image')
TF = pytest.importorskip('torchvision.transforms.functional')
transforms = pytest.importorskip('torchvision.transforms')

F32_ONE_UP = 1.0 + 2.0 ** -23


def _all_bytes3():
    c = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)


@pytest.mark.parametrize('factor', [0.0, 1.0, F32_ONE_UP, 0.6, 1.4, 0.7, 1.3, float(np.float32(0.6)),
                                    float(np.float32(1.4)), float(np.nextafter(np.float32(1.0), np.float32(0.0))),
                                    0.8137, 1.2999])
def test_blend_every_pair(factor):
    a, b = np.meshgrid(np.arange(256), np.arange(256), indexing='ij')
    A = np.repeat(a.astype(np.uint8)[..., None], 3, -1)
    B = np.repeat(b.astype(np.uint8)[..., None], 3, -1)
    want = np.array(Image.blend(Image.fromarray(A), Image.fromarray(B), factor))
    assert np.array_equal(P.blend(A, B, factor), want)


def test_conversions_every_input():
    img = _all_bytes3()
    assert np.array_equal(P.rgb_to_l(img), np.array(Image.fromarray(img).convert('L')))
    assert np.array_equal(P.rgb_to_hsv(img), np.array(Image.fromarray(img).convert('HSV')))
    assert np.array_equal(P.hsv_to_rgb(img), np.array(Image.fromarray(img, 'HSV').convert('RGB')))


@pytest.mark.parametrize('hue', [0.0, 0.159, -0.159, 0.3 / 3.14, -0.3 / 3.14, 0.5 / 3.14, -0.5 / 3.14,
                                 0.9 / 255, -0.9 / 255, 1 / 255, -1 / 255, 0.5, -0.5, 0.0037, -0.0037])
def test_hue_shift(hue):
    img = np.random.default_rng(1).integers(0, 256, (96, 128, 3), dtype=np.uint8)
    img[:8] = img[:8, :1]                                        # greys
    want = np.array(TF.adjust_hue(Image.fromarray(img), hue))
    assert np.array_equal(P.adjust_hue(img, P.hue_byte(hue)), want)
    assert P.hue_byte(hue) == int(np.int32(hue * 255).astype(np.uint8))
    if abs(hue) < 1 / 255:
        assert P.hue_byte(hue) == 0 and not np.array_equal(want, img)   # the round trip still runs


def test_contrast_mean_on_a_tie():
    img = np.zeros((1, 2, 3), np.uint8)
    img[0, 0], img[0, 1] = 100, 101                              # L = 100, 101: mean 100.5 -> 101
    assert P.contrast_mean(int(P.rgb_to_l(img).astype(np.int64).sum()), 2) == 101
    big = np.full((64, 64, 3), 37, np.uint8)
    big[:32] = 38                                                # mean 37.5 over 4096 pixels -> 38
    for x, f in ((img, 0.6137), (img, 1.37), (big, 0.0), (big, 1.31)):
        want = np.array(TF.adjust_contrast(Image.fromarray(x), f))
        assert np.array_equal(P.apply_op(x, P.CONTRAST, (1.0, f, 1.0), 0), want)
    assert np.all(P.apply_op(big, P.CONTRAST, (1.0, 0.0, 1.0), 0) == 38)


@pytest.mark.parametrize('order', list(itertools.permutations(range(4))))
def test_jitter_every_order(order):
    rng = np.random.default_rng(sum(o * 4 ** k for k, o in enumerate(order)))
    img = rng.integers(0, 256, (41, 67, 3), dtype=np.uint8)
    img[:10] = img[:10, :1]
    for _ in range(3):
        b, c, s = (float(np.float32(rng.uniform(0.6, 1.4))) for _ in range(3))
        h = float(np.float32(rng.uniform(-0.5 / 3.14, 0.5 / 3.14)))
        x = Image.fromarray(img)
        for op in order:
            x = [lambda y: TF.adjust_brightness(y, b), lambda y: TF.adjust_contrast(y, c),
                 lambda y: TF.adjust_saturation(y, s), lambda y: TF.adjust_hue(y, h)][op](x)
        assert np.array_equal(P.jitter(img, order, (b, c, s), h), np.array(x)), (order, b, c, s, h)
    # an op ColorJitter skips (strength 0: its factor is None)
    want = np.array(TF.adjust_saturation(TF.adjust_brightness(Image.fromarray(img), 0.75), 1.25))
    assert np.array_equal(P.jitter(img, (3, 0, 1, 2), (0.75, None, 1.25), None), want)


@pytest.mark.parametrize('strengths', [(0.4, 0.4, 0.4, 0.5 / 3.14), (0.3, 0.3, 0.3, 0.3 / 3.14), (0.4, 0, 0.2, 0),
                                       (0, 0.5, 0, 0.1)])
def test_parameter_stream_is_get_params(strengths):
    from tf_raft_b200.datasets.augmentor import jitter_params
    cj = transforms.ColorJitter(*strengths)
    for seed in range(20):
        torch.manual_seed(seed)
        fn_idx, *factors = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
        want = (tuple(int(i) for i in fn_idx), *factors)
        torch.manual_seed(seed)
        assert jitter_params(*strengths) == want
        assert all(f is None or float(np.float32(f)) == f for f in want[1:])   # float32 draws: exact as blend's


class _Recording(transforms.ColorJitter):
    def __init__(self, *args):
        super().__init__(*args)
        self.drawn = []

    def get_params(self, *ranges):
        fn_idx, *factors = transforms.ColorJitter.get_params(*ranges)
        self.drawn.append((tuple(int(i) for i in fn_idx), *factors))
        return (fn_idx, *factors)


def _seed_with_gate(asym):
    for seed in range(1000):
        np.random.seed(seed)
        if (np.random.rand() < 0.2) == asym:
            return seed
    raise AssertionError('no seed')


@pytest.mark.parametrize('kind,asym', [('dense', False), ('dense', True), ('sparse', False)])
def test_sample_params_follows_raft(kind, asym):
    """The GPU augmentor's sampler and RAFT's augmentor, seeded alike, draw the same jitter parameters (both gate
    outcomes for FlowAugmentor) and leave np.random and torch's generator in the same state."""
    from oracle import raft_augment as R
    from tf_raft_b200.datasets import FlowAugmentor, SparseFlowAugmentor
    h, w, crop = 120, 176, (64, 96)
    rng = np.random.default_rng(3)
    img1, img2 = (rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(2))
    flow = rng.standard_normal((h, w, 2)).astype(np.float32)
    valid = (rng.uniform(size=(h, w)) < 0.5).astype(np.float32)
    seed = _seed_with_gate(asym)
    for torch_seed in (0, 7):
        ours = (FlowAugmentor if kind == 'dense' else SparseFlowAugmentor)(crop, colour='torchvision', device='cpu')
        ref = (R.FlowAugmentor if kind == 'dense' else R.SparseFlowAugmentor)(crop)
        ref.photo_aug = _Recording(*((0.4, 0.4, 0.4, 0.5 / 3.14) if kind == 'dense' else (0.3, 0.3, 0.3, 0.3 / 3.14)))
        np.random.seed(seed)
        torch.manual_seed(torch_seed)
        p = ours.sample_params(h, w)
        states = np.random.get_state()[1].copy(), torch.get_rng_state()
        np.random.seed(seed)
        torch.manual_seed(torch_seed)
        ref(img1, img2, flow) if kind == 'dense' else ref(img1, img2, flow, valid)
        assert p.jitter == tuple(ref.photo_aug.drawn)
        assert len(p.jitter) == (2 if asym else 1)
        assert p.colour1 == p.colour2 == (None, None)
        assert np.array_equal(states[0], np.random.get_state()[1]) and torch.equal(states[1], torch.get_rng_state())


def test_default_sampler_draws_no_torch_and_options_are_checked():
    from tf_raft_b200.datasets import AugmentParams, FlowAugmentor, SparseFlowAugmentor
    torch.manual_seed(5)
    before = torch.get_rng_state()
    np.random.seed(2)
    p = FlowAugmentor((64, 96), device='cpu').sample_params(120, 176)
    assert p.jitter == () and torch.equal(before, torch.get_rng_state())
    assert AugmentParams(*[None] * 11).jitter == ()
    for cls in (FlowAugmentor, SparseFlowAugmentor):
        with pytest.raises(ValueError, match='colour'):
            cls((64, 96), colour='PIL', device='cpu')
