"""The convolutions train_precision='f16x2' puts on the tensor cores, derived from the parameter shapes of both variants'
layers, as the training graph (tf_raft_b200/train.py TrainGraph) applies them, and the sizes they run at."""
import re

ELIGIBLE_MIN_CIN = 64        # TrainGraph._conv_f16x2


def _layer_params(variant):
    from tf_raft_b200 import layers
    if variant == 'raft':
        enc = {'fnet': layers.BasicEncoder(output_dim=256, norm_type='instance', device='cpu', seed=0),
               'cnet': layers.BasicEncoder(output_dim=256, norm_type='batch', device='cpu', seed=0)}
        upd = layers.BasicUpdateBlock(filters=128, device='cpu', seed=0)
    else:
        enc = {'fnet': layers.SmallEncoder(output_dim=128, norm_type='instance', device='cpu', seed=0),
               'cnet': layers.SmallEncoder(output_dim=160, norm_type=None, device='cpu', seed=0)}
        upd = layers.SmallUpdateBlock(filters=96, device='cpu', seed=0)
    out = {}
    for prefix, e in enc.items():
        out.update({f'{prefix}.{k}': v for k, v in e.params.items()})
    out.update({f'update_block.{k}': v for k, v in upd.params.items()})
    return out


def _stride_padding(name, variant):
    """(stride, padding) TrainGraph.conv applies to the kernel `name` (encoder / res_block / update_block)."""
    if re.fullmatch(r'(fnet|cnet)\.conv1', name):
        return 2, 'same'
    m = re.fullmatch(r'(fnet|cnet)\.layer(\d)\.(\d)\.(conv1|conv2|downsample\.0)', name)
    if m:
        first_of_stage = int(m.group(2)) > 1 and m.group(3) == '0'
        if m.group(4) == 'downsample.0':
            return 2, 'valid'
        return (2 if first_of_stage and m.group(4) == 'conv1' else 1), 'same'
    if re.fullmatch(r'(fnet|cnet)\.conv2', name) or name.endswith('mask.2'):
        return 1, 'valid'
    if name.endswith('encoder.convc1') and variant == 'raft':
        return 1, 'valid'
    return 1, 'same'


def _stage(name):
    """Resolution divisor and batch multiplier (fnet runs on both images) of the layer."""
    m = re.match(r'(fnet|cnet)\.(?:layer(\d)|conv(\d))', name)
    if not m:
        return 8, 1
    div = {1: 2, 2: 4, 3: 8}[int(m.group(2))] if m.group(2) else (2 if m.group(3) == '1' else 8)
    return div, (2 if m.group(1) == 'fnet' else 1)


def layers(variant):
    """[(name, cin, kh, kw, cout, stride, padding, div, batch_mult, eligible)] for every convolution of the variant."""
    out = []
    for k, v in _layer_params(variant).items():
        if not k.endswith('.kernel'):
            continue
        name = k[:-len('.kernel')]
        kh, kw, cin, cout = v.shape
        stride, padding = _stride_padding(name, variant)
        div, bm = _stage(name)
        eligible = stride == 1 and cin >= ELIGIBLE_MIN_CIN and kh % 2 == 1 and kw % 2 == 1 and \
            (padding == 'same' or kh == kw == 1)
        out.append((name, int(cin), int(kh), int(kw), int(cout), stride, padding, div, bm, eligible))
    return out


def shapes(variant):
    """Distinct eligible (cin, kh, kw, cout, div, batch_mult) of the variant."""
    return sorted({(c, kh, kw, co, d, bm) for _, c, kh, kw, co, _, _, d, bm, e in layers(variant) if e})


# (name, batch, image H, image W): Chairs training crops (batch 4, 368 x 496), Sintel (368 x 768) and a ragged size
# whose feature maps are no tile multiples.
SIZES = (('chairs', 4, 368, 496), ('sintel', 1, 368, 768), ('ragged', 2, 296, 424))


def cases():
    """[(id, B, H, W, cin, kh, kw, cout)] of every eligible shape of both variants at every size in SIZES."""
    out = set()
    for variant in ('raft', 'small'):
        for c, kh, kw, co, div, bm in shapes(variant):
            for size, b, H, W in SIZES:
                out.add((f'{size}-{b * bm}x{H // div}x{W // div}-{c}-{kh}x{kw}-{co}', b * bm, H // div, W // div, c, kh, kw,
                         co))
    return sorted(out)
