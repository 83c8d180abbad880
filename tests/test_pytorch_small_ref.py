"""The original PyTorch RAFT-small on the CPU: a module transcription of its architecture pins the layout of
`synthetic_small_checkpoint` and agrees with the oracle's `forward_small`; the loader maps such a file and refuses the
other model's; `upflow8_emulated` against float64 F.interpolate(align_corners=True).  No GPU needed."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import raft_pytorch as rp, raft_pytorch_small as rps, weights
from tf_raft_b200.checkpoint import _pt_instance_norms, load_pytorch_checkpoint, to_pytorch_state_dict

F32 = np.float32


# ----------------------------------------------------------------------------- the architecture as nn.Modules
class BottleneckBlock(nn.Module):
    def __init__(self, in_planes, planes, norm_fn, stride=1):
        super().__init__()
        self.conv1 = nn.Conv2d(in_planes, planes // 4, kernel_size=1, padding=0)
        self.conv2 = nn.Conv2d(planes // 4, planes // 4, kernel_size=3, padding=1, stride=stride)
        self.conv3 = nn.Conv2d(planes // 4, planes, kernel_size=1, padding=0)
        self.relu = nn.ReLU()

        def norm(c):
            return nn.InstanceNorm2d(c) if norm_fn == 'instance' else nn.Sequential()
        self.norm1, self.norm2, self.norm3 = norm(planes // 4), norm(planes // 4), norm(planes)
        self.downsample = None
        if stride != 1:
            self.norm4 = norm(planes)
            self.downsample = nn.Sequential(nn.Conv2d(in_planes, planes, kernel_size=1, stride=stride), self.norm4)

    def forward(self, x):
        y = self.relu(self.norm1(self.conv1(x)))
        y = self.relu(self.norm2(self.conv2(y)))
        y = self.relu(self.norm3(self.conv3(y)))
        if self.downsample is not None:
            x = self.downsample(x)
        return self.relu(x + y)


class SmallEncoder(nn.Module):
    def __init__(self, output_dim, norm_fn):
        super().__init__()
        self.norm1 = nn.InstanceNorm2d(32) if norm_fn == 'instance' else nn.Sequential()
        self.conv1 = nn.Conv2d(3, 32, kernel_size=7, stride=2, padding=3)
        self.relu1 = nn.ReLU()
        self.in_planes = 32
        self.layer1 = self._layer(32, norm_fn, 1)
        self.layer2 = self._layer(64, norm_fn, 2)
        self.layer3 = self._layer(96, norm_fn, 2)
        self.conv2 = nn.Conv2d(96, output_dim, kernel_size=1)

    def _layer(self, dim, norm_fn, stride):
        layers = (BottleneckBlock(self.in_planes, dim, norm_fn, stride), BottleneckBlock(dim, dim, norm_fn, 1))
        self.in_planes = dim
        return nn.Sequential(*layers)

    def forward(self, x):
        x = self.relu1(self.norm1(self.conv1(x)))
        return self.conv2(self.layer3(self.layer2(self.layer1(x))))


class SmallMotionEncoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.convc1 = nn.Conv2d(196, 96, 1, padding=0)
        self.convf1 = nn.Conv2d(2, 64, 7, padding=3)
        self.convf2 = nn.Conv2d(64, 32, 3, padding=1)
        self.conv = nn.Conv2d(128, 80, 3, padding=1)

    def forward(self, flow, corr):
        cor = F.relu(self.convc1(corr))
        flo = F.relu(self.convf2(F.relu(self.convf1(flow))))
        return torch.cat([F.relu(self.conv(torch.cat([cor, flo], dim=1))), flow], dim=1)


class ConvGRU(nn.Module):
    def __init__(self, hidden_dim=96, input_dim=146):
        super().__init__()
        self.convz = nn.Conv2d(hidden_dim + input_dim, hidden_dim, 3, padding=1)
        self.convr = nn.Conv2d(hidden_dim + input_dim, hidden_dim, 3, padding=1)
        self.convq = nn.Conv2d(hidden_dim + input_dim, hidden_dim, 3, padding=1)

    def forward(self, h, x):
        hx = torch.cat([h, x], dim=1)
        z, r = torch.sigmoid(self.convz(hx)), torch.sigmoid(self.convr(hx))
        q = torch.tanh(self.convq(torch.cat([r * h, x], dim=1)))
        return (1 - z) * h + z * q


class FlowHead(nn.Module):
    def __init__(self, input_dim=96, hidden_dim=128):
        super().__init__()
        self.conv1 = nn.Conv2d(input_dim, hidden_dim, 3, padding=1)
        self.conv2 = nn.Conv2d(hidden_dim, 2, 3, padding=1)

    def forward(self, x):
        return self.conv2(F.relu(self.conv1(x)))


class SmallUpdateBlock(nn.Module):
    def __init__(self):
        super().__init__()
        self.encoder = SmallMotionEncoder()
        self.gru = ConvGRU(96, 82 + 64)
        self.flow_head = FlowHead(96, 128)

    def forward(self, net, inp, corr, flow):
        net = self.gru(net, torch.cat([inp, self.encoder(flow, corr)], dim=1))
        return net, None, self.flow_head(net)


class RAFTSmall(nn.Module):
    def __init__(self):
        super().__init__()
        self.fnet = SmallEncoder(128, 'instance')
        self.cnet = SmallEncoder(160, 'none')
        self.update_block = SmallUpdateBlock()

    @staticmethod
    def _sample(img, coords):
        H, W = img.shape[-2:]
        x, y = coords.split([1, 1], dim=-1)
        grid = torch.cat([2 * x / (W - 1) - 1, 2 * y / (H - 1) - 1], dim=-1)
        return F.grid_sample(img, grid, align_corners=True)

    def forward(self, image1, image2, iters):
        image1, image2 = 2 * (image1 / 255.0) - 1.0, 2 * (image2 / 255.0) - 1.0
        fmap1, fmap2 = self.fnet(torch.cat([image1, image2])).split(image1.shape[0])
        b, c, h, w = fmap1.shape
        corr = torch.matmul(fmap1.view(b, c, h * w).transpose(1, 2), fmap2.view(b, c, h * w)) / c ** 0.5
        pyr = [corr.reshape(b * h * w, 1, h, w)]
        for _ in range(3):
            pyr.append(F.avg_pool2d(pyr[-1], 2, stride=2))
        net, inp = torch.split(self.cnet(image1), [96, 64], dim=1)
        net, inp = torch.tanh(net), torch.relu(inp)
        ys, xs = torch.meshgrid(torch.arange(h, dtype=image1.dtype), torch.arange(w, dtype=image1.dtype), indexing='ij')
        coords0 = torch.stack([xs, ys])[None].repeat(b, 1, 1, 1)
        coords1 = coords0.clone()
        d = torch.linspace(-3, 3, 7, dtype=image1.dtype)
        delta = torch.stack(torch.meshgrid(d, d, indexing='ij'), dim=-1).view(1, 7, 7, 2)
        preds = []
        for _ in range(iters):
            cc = coords1.permute(0, 2, 3, 1).reshape(b * h * w, 1, 1, 2)
            corr = torch.cat([self._sample(p, cc / 2 ** i + delta).view(b, h, w, -1) for i, p in enumerate(pyr)], dim=-1)
            net, _, dflow = self.update_block(net, inp, corr.permute(0, 3, 1, 2), coords1 - coords0)
            coords1 = coords1 + dflow
            flow = coords1 - coords0
            preds.append(8 * F.interpolate(flow, size=(8 * h, 8 * w), mode='bilinear', align_corners=True))
        return preds


@pytest.fixture(scope='module')
def ckpt():
    return rps.synthetic_small_checkpoint(seed=11)


def _model_expect():
    import tf_raft_b200 as T
    return T.SmallRAFT(conventions='pytorch', blocks='bottleneck', device='cpu').state_dict()


def test_module_transcription_loads_the_synthetic_layout_and_equals_the_oracle(ckpt):
    """load_state_dict(strict=True) pins the key set and shapes; the fp64 forward equals forward_small to 1e-12."""
    model = RAFTSmall().double().eval()
    model.load_state_dict({k[len('module.'):]: v for k, v in ckpt.items()}, strict=True)
    rng = np.random.default_rng(2)
    im1 = rng.uniform(0, 255, (2, 128, 144, 3))            # every pyramid level at least 2 x 2
    im2 = np.clip(im1 + rng.normal(0, 20, im1.shape), 0, 255)
    with torch.no_grad():
        got = model(torch.from_numpy(im1).permute(0, 3, 1, 2), torch.from_numpy(im2).permute(0, 3, 1, 2), iters=3)
    want, _ = rps.forward_small(ckpt, im1, im2, iters=3)
    for g, w in zip(got, want):
        np.testing.assert_allclose(g.permute(0, 2, 3, 1).numpy(), w, rtol=0, atol=1e-12)
    assert float(np.abs(want[-1]).max()) > 0.1                 # the flows are not trivially zero


def test_loader_maps_raft_small_and_round_trips(ckpt, tmp_path):
    expect = _model_expect()
    path = tmp_path / 'raft-small-synthetic.pth'
    torch.save(ckpt, path)
    params = load_pytorch_checkpoint(str(path), expect=expect)
    assert set(params) == set(expect)
    for k, v in params.items():
        assert v.dtype == np.float32 and v.shape == tuple(expect[k].shape), k
    sd = {k[len('module.'):]: v.numpy() for k, v in ckpt.items()}
    for name in ('fnet.conv1', 'fnet.layer2.0.conv2', 'cnet.layer3.0.downsample.0', 'fnet.layer1.1.conv3',
                 'update_block.gru.convq', 'update_block.encoder.convf1'):
        np.testing.assert_array_equal(params[name + '.kernel'], sd[name + '.weight'].transpose(2, 3, 1, 0))
        np.testing.assert_array_equal(params[name + '.bias'], sd[name + '.bias'])
    # identity affine for every fnet instance norm, at the widths of the architecture; nothing for cnet
    norms = dict(_pt_instance_norms(small=True))
    assert len(norms) == 1 + 6 * 3 + 2
    assert norms['fnet.norm1'] == 32 and norms['fnet.layer1.0.norm1'] == 8 and norms['fnet.layer2.1.norm2'] == 16
    assert norms['fnet.layer3.0.norm3'] == 96 and norms['fnet.layer3.0.downsample.1'] == 96
    for name, c in norms.items():
        np.testing.assert_array_equal(params[name + '.gamma'], np.ones(c, F32))
        np.testing.assert_array_equal(params[name + '.beta'], np.zeros(c, F32))
    assert not any(k.startswith('cnet.') and ('norm' in k or 'downsample.1' in k) for k in params)
    # the writer gives raft-small.pth's keys and bytes back, with no norm entries
    out = to_pytorch_state_dict(params)
    assert set(out) == set(ckpt)
    for k, v in ckpt.items():
        assert out[k].dtype == torch.float32 and torch.equal(out[k], v), k
    again = load_pytorch_checkpoint({k[len('module.'):]: v for k, v in ckpt.items()}, expect=expect)
    assert all(np.array_equal(again[k], params[k]) for k in params)


def test_loader_refuses_the_other_model_by_name(ckpt):
    small_expect = _model_expect()
    basic_expect = {k: np.zeros(s, F32) for k, s in weights.param_shapes('raft').items()}
    with pytest.raises(ValueError, match='RAFT-small') as e:
        load_pytorch_checkpoint(ckpt, expect=basic_expect)
    assert 'conv3' in str(e.value)
    with pytest.raises(ValueError, match='RAFT-small'):
        load_pytorch_checkpoint(rp.synthetic_checkpoint(seed=1), expect=small_expect)
    # a RAFT-small file with a layer missing or mis-shaped is reported like any other
    sd = dict(ckpt)
    del sd['module.fnet.layer2.0.conv3.bias']
    sd['module.cnet.conv2.weight'] = torch.zeros(128, 96, 1, 1)
    with pytest.raises(ValueError) as e:
        load_pytorch_checkpoint(sd, expect=small_expect)
    assert 'fnet.layer2.0.conv3.bias' in str(e.value) and 'cnet.conv2.kernel' in str(e.value)


def test_the_basic_model_loads_as_before():
    """The basic model's mapping is unchanged: the same parameters from the same file."""
    basic_expect = {k: np.zeros(s, F32) for k, s in weights.param_shapes('raft').items()}
    params = load_pytorch_checkpoint(rp.synthetic_checkpoint(seed=4), expect=basic_expect)
    assert set(params) == set(basic_expect)
    np.testing.assert_array_equal(params['fnet.layer2.0.downsample.1.gamma'], np.ones(96, F32))


def _axis_positions(n):
    """The emulation's per-axis float32 source positions, and the exact ones."""
    scale = F32(F32(n - 1) / F32(8 * n - 1))
    X = np.arange(8 * n)
    return (scale * X.astype(F32)).astype(F32), X * (n - 1) / (8 * n - 1)


@pytest.mark.parametrize('shape', [(1, 1, 1), (2, 1, 5), (1, 6, 1), (1, 7, 3), (2, 17, 30), (1, 55, 128)])
def test_upflow8_emulated_against_fp64_interpolate(shape):
    """The emulation equals fp64 bilinear interpolation at its own float32 source positions to 4 ulps of the output's
    scale; those positions are within 1 ulp of the exact ones, so against fp64 F.interpolate it is within 8 * the
    largest neighbour difference * that position error, plus the same 4 ulps."""
    b, h, w = shape
    rng = np.random.default_rng(h * 100 + w)
    flow = (rng.standard_normal((b, h, w, 2)) * 6).astype(F32)
    got = rps.upflow8_emulated(flow)
    assert got.shape == (b, 8 * h, 8 * w, 2) and got.dtype == F32
    ref = (8 * F.interpolate(torch.from_numpy(flow).double().permute(0, 3, 1, 2), size=(8 * h, 8 * w), mode='bilinear',
                             align_corners=True)).permute(0, 2, 3, 1).numpy()
    scale = float(np.abs(ref).max())
    pos_err = 0.0
    for n in (h, w):
        src, exact = _axis_positions(n)
        err = np.abs(src.astype(np.float64) - exact)
        assert np.all(err <= np.spacing(np.maximum(src, F32(1e-30)).astype(F32)) + 1e-300), n
        pos_err = max(pos_err, float(err.max()))
    f = flow.astype(np.float64)
    at_own = rps.upflow8_fp32_positions(flow)
    ulp = np.spacing(F32(scale))
    assert float(np.abs(got - at_own).max()) <= 4 * ulp
    diff = max(float(np.abs(np.diff(f, axis=a)).max()) if f.shape[a] > 1 else 0.0 for a in (1, 2))
    assert float(np.abs(got - ref).max()) <= 8 * 2 * diff * pos_err + 4 * ulp
    if h == 1 and w == 1:                                    # a single cell is copied, times 8 exactly
        np.testing.assert_array_equal(got, np.broadcast_to(8 * flow, got.shape))
