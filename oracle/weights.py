"""Deterministic parameter generator for RAFT / SmallRAFT (test infrastructure).

The reference's checkpoints live on GCS only (README.md:69-90) and TF's RNG
stream is not reproducible without TF, so tests draw parameters from NumPy's
PCG64 with the Keras default *distributions*: `glorot_uniform` kernels
(limit sqrt(6/(fan_in+fan_out)), fan = kh*kw*C), zero biases, gamma 1 / beta 0,
BatchNorm moving mean 0 / variance 1 (SURVEY.md Appendix A).  `bias_scale` and
`norm_jitter` perturb the zero/one defaults so that parity tests also exercise
the bias / affine / moving-statistics code paths.

Names are the Keras attribute paths of the reference (SURVEY.md Appendix B):
kernels are HWIO `(kh, kw, Cin, Cout)` float32.
"""
from collections import OrderedDict

import numpy as np

F32 = np.float32


def _norm_entries(prefix, norm_type, c):
    if norm_type == 'instance':      # tfa.layers.InstanceNormalization (extractor.py:12)
        return [(prefix + '.gamma', (c,)), (prefix + '.beta', (c,))]
    if norm_type == 'batch':         # layers.BatchNormalization (extractor.py:10)
        return [(prefix + '.gamma', (c,)), (prefix + '.beta', (c,)),
                (prefix + '.moving_mean', (c,)), (prefix + '.moving_variance', (c,))]
    if norm_type is None:            # layers.Lambda identity (extractor.py:14)
        return []
    raise ValueError(f'Invalid norm_type specified: {norm_type}')


def _conv_entries(prefix, kh, kw, cin, cout):
    return [(prefix + '.kernel', (kh, kw, cin, cout)), (prefix + '.bias', (cout,))]


def encoder_shapes(prefix, norm_type, c0, stages, out_dim):
    """extractor.py:88-130 (Basic: c0=64, stages 64/96/128) and :133-175 (Small: 32, 32/64/96)."""
    e = _conv_entries(prefix + '.conv1', 7, 7, 3, c0) + _norm_entries(prefix + '.norm1', norm_type, c0)
    cin = c0
    for li, (c, s) in enumerate(stages, start=1):
        for bi, stride in enumerate((s, 1)):
            p = f'{prefix}.layer{li}.{bi}'
            e += _conv_entries(p + '.conv1', 3, 3, cin, c) + _conv_entries(p + '.conv2', 3, 3, c, c)
            e += _norm_entries(p + '.norm1', norm_type, c) + _norm_entries(p + '.norm2', norm_type, c)
            if stride != 1:          # extractor.py:33-39
                e += _conv_entries(p + '.downsample.0', 1, 1, cin, c)
                e += _norm_entries(p + '.downsample.1', norm_type, c)
            cin = c
    e += _conv_entries(prefix + '.conv2', 1, 1, cin, out_dim)
    return e


def basic_update_shapes(prefix='update_block', corr_ch=324, hidden=128):
    """update.py:128-141 with BasicMotionEncoder :88-95, SepConvGRU :38-49, FlowHead :5-11."""
    e = []
    e += _conv_entries(prefix + '.encoder.convc1', 1, 1, corr_ch, 256)
    e += _conv_entries(prefix + '.encoder.convc2', 3, 3, 256, 192)
    e += _conv_entries(prefix + '.encoder.convf1', 7, 7, 2, 128)
    e += _conv_entries(prefix + '.encoder.convf2', 3, 3, 128, 64)
    e += _conv_entries(prefix + '.encoder.conv', 3, 3, 256, 126)
    gin = hidden + 128 + 128
    for n in ('convz1', 'convr1', 'convq1'):
        e += _conv_entries(f'{prefix}.gru.{n}', 1, 5, gin, hidden)
    for n in ('convz2', 'convr2', 'convq2'):
        e += _conv_entries(f'{prefix}.gru.{n}', 5, 1, gin, hidden)
    e += _conv_entries(prefix + '.flow_head.conv1', 3, 3, hidden, 256)
    e += _conv_entries(prefix + '.flow_head.conv2', 3, 3, 256, 2)
    e += _conv_entries(prefix + '.mask.0', 3, 3, hidden, 256)
    e += _conv_entries(prefix + '.mask.2', 1, 1, 256, 576)
    return e


def small_update_shapes(prefix='update_block', corr_ch=196, hidden=96):
    """update.py:109-116 with SmallMotionEncoder :70-76, ConvGRU :17-24, FlowHead(128)."""
    e = []
    e += _conv_entries(prefix + '.encoder.convc1', 1, 1, corr_ch, 96)
    e += _conv_entries(prefix + '.encoder.convf1', 7, 7, 2, 64)
    e += _conv_entries(prefix + '.encoder.convf2', 3, 3, 64, 32)
    e += _conv_entries(prefix + '.encoder.conv', 3, 3, 128, 80)
    gin = hidden + 64 + 82
    for n in ('convz', 'convr', 'convq'):
        e += _conv_entries(f'{prefix}.gru.{n}', 3, 3, gin, hidden)
    e += _conv_entries(prefix + '.flow_head.conv1', 3, 3, hidden, 128)
    e += _conv_entries(prefix + '.flow_head.conv2', 3, 3, 128, 2)
    return e


def param_shapes(variant):
    """Full parameter tree of RAFT (model.py:24-30) or SmallRAFT (model.py:182-188)."""
    if variant == 'raft':
        e = encoder_shapes('fnet', 'instance', 64, [(64, 1), (96, 2), (128, 2)], 256)
        e += encoder_shapes('cnet', 'batch', 64, [(64, 1), (96, 2), (128, 2)], 256)
        e += basic_update_shapes()
    elif variant == 'small':
        e = encoder_shapes('fnet', 'instance', 32, [(32, 1), (64, 2), (96, 2)], 128)
        e += encoder_shapes('cnet', None, 32, [(32, 1), (64, 2), (96, 2)], 160)
        e += small_update_shapes()
    else:
        raise ValueError(variant)
    return OrderedDict(e)


def init_params(variant, seed=1234, bias_scale=0.0, norm_jitter=0.0):
    """name -> float32 ndarray, drawn in tree order from default_rng(seed)."""
    return draw_params(param_shapes(variant), seed, bias_scale, norm_jitter)


def draw_params(shapes, seed=1234, bias_scale=0.0, norm_jitter=0.0):
    """{name: shape} (in order) -> name -> float32 ndarray, with the distributions of the module docstring."""
    rng = np.random.default_rng(seed)
    out = OrderedDict()
    for name, shape in OrderedDict(shapes).items():
        leaf = name.rsplit('.', 1)[1]
        if leaf == 'kernel':
            kh, kw, cin, cout = shape
            limit = np.sqrt(6.0 / (kh * kw * cin + kh * kw * cout))
            v = rng.uniform(-limit, limit, shape)
        elif leaf == 'bias':
            v = rng.uniform(-bias_scale, bias_scale, shape) if bias_scale else np.zeros(shape)
        elif leaf in ('gamma', 'moving_variance'):
            v = 1.0 + (rng.uniform(-norm_jitter, norm_jitter, shape) if norm_jitter else 0.0) * np.ones(shape)
        elif leaf in ('beta', 'moving_mean'):
            v = rng.uniform(-norm_jitter, norm_jitter, shape) if norm_jitter else np.zeros(shape)
        else:
            raise KeyError(name)
        out[name] = np.ascontiguousarray(v, dtype=F32)
    return out


def n_params(variant, trainable_only=True):
    n = 0
    for name, shape in param_shapes(variant).items():
        if trainable_only and name.rsplit('.', 1)[1].startswith('moving_'):
            continue
        n += int(np.prod(shape))
    return n
