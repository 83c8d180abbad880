"""The concurrent inference encode (raft_b200_encode_pair, RAFT._encode_pair) against the serial one, bit for bit.

RAFT._encode_pair runs fnet(image1), fnet(image2) and cnet(image1) as concurrent branches.  Every encoder kernel treats
each image on its own, so its outputs, and the correlation pyramid built from them, must equal those of the separate
fnet([image1, image2]) / cnet / context_split calls exactly: eagerly, on a non-default caller stream, and captured into
a CUDA graph that is replayed on two different inputs.
"""
import numpy as np
import pytest
import torch

import cases
from oracle import weights

pytestmark = pytest.mark.gpu
SHAPES = [(4, 448, 512), (4, 448, 1024), (1, 448, 512), (4, 440, 1016)]


@pytest.fixture(scope='module', params=['raft', 'small'])
def model(request):
    import tf_raft_b200 as T
    from tf_raft_b200 import _lib
    assert _lib.lib().raft_b200_device_ok(torch.cuda.current_device()) == 0, 'needs an sm_90 GPU'
    m = (T.RAFT if request.param == 'raft' else T.SmallRAFT)(iters=2, iters_pred=2, precision='f16x2')
    m.load_params(weights.init_params(request.param, 7, bias_scale=0.05, norm_jitter=0.1))
    return m


def with_pyramid(model, fmap1, fmap2, net, inp):
    from tf_raft_b200 import CorrBlock
    cb = CorrBlock(fmap1, fmap2, num_levels=model.corr_levels, radius=model.corr_radius, precision=model.precision)
    return [fmap1, fmap2, net, inp] + cb.corr_pyramid


def serial(model, a, b):
    fmap1, fmap2 = model.fnet([a, b], training=False, raw_image=True)
    return with_pyramid(model, fmap1, fmap2, *model._context(a, False))


def concurrent(model, a, b):
    return with_pyramid(model, *model._encode_pair(a, b))


def assert_equal(got, want, what):
    names = ['fmap1', 'fmap2', 'net', 'inp'] + [f'pyramid level {l}' for l in range(len(want) - 4)]
    for name, g, w in zip(names, got, want):
        assert g.shape == w.shape, f'{what}: {name} shape {tuple(g.shape)} != {tuple(w.shape)}'
        assert torch.equal(g, w), f'{what}: {name} differs, max-abs {float((g - w).abs().max()):.3e}'


def inputs(B, H, W, seed):
    return [torch.from_numpy(x).cuda() for x in cases.images(B, H, W, seed, seed + 1)]


@pytest.mark.parametrize('B,H,W', SHAPES, ids=lambda v: str(v))
def test_concurrent_encode_equals_serial(model, B, H, W):
    a, b = inputs(B, H, W, 10)
    want = serial(model, a, b)
    assert_equal(concurrent(model, a, b), want, 'eager')
    torch.cuda.synchronize()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = concurrent(model, a, b)
    torch.cuda.current_stream().wait_stream(side)
    assert_equal(got, want, 'non-default caller stream')

    a2, b2 = inputs(B, H, W, 20)
    want2 = serial(model, a2, b2)
    sa, sb = a.clone(), b.clone()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = concurrent(model, sa, sb)
    graph.replay()
    assert_equal(outs, want, 'graph replay 1')
    sa.copy_(a2)
    sb.copy_(b2)
    graph.replay()
    assert_equal(outs, want2, 'graph replay 2 (new inputs)')
    torch.cuda.synchronize()


def test_forward_equals_serial_encode(model):
    """The whole inference forward on the concurrent encode gives the final flow of the serial encode, bit for bit."""
    B, H, W = 4, 448, 512
    a, b = inputs(B, H, W, 30)
    got = model([a, b], training=False, last_only=True)[-1]
    fmap1, fmap2 = model.fnet([a, b], training=False, raw_image=True)
    net, inp = model._context(a, False)
    want = model._iterate(fmap1, fmap2, net, inp, B, H, W, False, True, None)[-1]
    assert torch.equal(got, want), float((got - want).abs().max())
    assert np.isfinite(got.cpu().numpy()).all()
