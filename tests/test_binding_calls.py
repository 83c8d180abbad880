"""The package reaches libraft_b200.so through `_lib.call` (stream-taking entry points) and `_lib.query_bytes` (size
queries) only, so no call site can pair one device's pointers with another device's stream; the layers' workspace
caches keep one shape; and the shared parameter store draws the seeded default weights it always drew."""
import ast
import ctypes
import glob
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import corr_np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
# entry points with neither a stream nor a single size_t result: called directly on `_lib.lib()`
DIRECT = {'strerror', 'abi_version', 'device_ok', 'launch_count', 'launch_count_reset', 'profile_loop', 'profile_read',
          'corr_pyramid_sizes'}


def _entry_points():
    from tf_raft_b200 import _lib
    streamed, sized = set(), set()
    for symbol, (_, args) in _lib._SIGNATURES.items():
        name = symbol[len('raft_b200_'):]
        if name in DIRECT:
            continue
        if args[-1] is ctypes.c_void_p:
            streamed.add(name)
        elif args[-1] is ctypes.POINTER(ctypes.c_size_t):
            sized.add(name)
        else:
            raise AssertionError(f'{symbol}: neither stream-taking, a size query, nor listed in DIRECT')
    return streamed, sized


def test_every_entry_point_is_classified():
    streamed, sized = _entry_points()
    assert {'upflow8', 'bilinear_sampler', 'forward_loop', 'encode_pair', 'augment_dense'} <= streamed
    assert sized == {'corr_workspace_bytes', 'augment_workspace_bytes', 'flow_metrics_workspace_bytes',
                     'update_prepared_bytes', 'update_workspace_bytes', 'encoder_prepared_bytes',
                     'encoder_workspace_bytes', 'encode_pair_workspace_bytes'}


def test_no_module_binds_a_stream_or_a_size_query_by_hand():
    streamed, sized = _entry_points()
    files = glob.glob(os.path.join(ROOT, 'tf_raft_b200', '**', '*.py'), recursive=True)
    assert len(files) > 10
    bad = []
    for path in files:
        rel = os.path.relpath(path, ROOT)
        if rel == os.path.join('tf_raft_b200', '_lib.py'):
            continue
        for node in ast.walk(ast.parse(open(path).read(), path)):
            if not isinstance(node, ast.Attribute):
                continue
            if node.attr.startswith('raft_b200_') and node.attr[len('raft_b200_'):] in streamed | sized:
                bad.append(f'{rel}:{node.lineno}: .{node.attr} -- use _lib.call / _lib.query_bytes')
            if node.attr == 'stream' and isinstance(node.value, ast.Name) and node.value.id == '_lib':
                bad.append(f'{rel}:{node.lineno}: _lib.stream -- _lib.call passes the stream')
    assert not bad, '\n'.join(bad)


def test_query_bytes_returns_the_size_and_names_the_query_on_error():
    from tf_raft_b200 import build, _lib
    build.build()
    assert _lib.query_bytes('update_workspace_bytes', 0, 4, 56, 64, 1) > 0
    with pytest.raises(RuntimeError) as err:
        _lib.query_bytes('update_workspace_bytes', 7, 4, 56, 64, 1)
    assert str(err.value) == 'raft_b200 update_workspace_bytes failed: [-1] ' + _lib.strerror(-1)


def test_workspace_cache_keeps_one_shape_and_sizes_on_a_miss_only():
    from tf_raft_b200 import _lib
    cache, asked = _lib.WorkspaceCache(), []

    def nbytes(n):
        return lambda: asked.append(n) or n

    assert cache.buffers() == []
    a = cache.get((1, 8, 8), 'cpu', nbytes(64))
    assert a.dtype == torch.uint8 and a.numel() == 64 and asked == [64]
    assert cache.get((1, 8, 8), 'cpu', nbytes(999)) is a and asked == [64]           # a hit asks nothing
    b = cache.get((2, 8, 8), 'cpu', nbytes(128))
    assert b.numel() == 128 and asked == [64, 128]
    assert [t is b for t in cache.buffers()] == [True]                               # the first shape's buffer is dropped
    assert cache.get((1, 8, 8), 'cpu', nbytes(64)) is not a and asked == [64, 128, 64]


# SHA-256 over names and bytes of the default parameters at seeds 0 and 3 (the encoders at each norm type)
SEEDED = {
    'BasicEncoder': '2a07dbfdbb6af87220952cd34deb0a6f680e14571ea530f631e3bfac27b04c7b',
    'SmallEncoder': 'a66e92e80836f43d0d87ab3f810102563189bb7f3b0060aeaf9bde2f56f29914',
    'BasicUpdateBlock': 'e5541174348626e3c751a03f2bd8f0960496f06960de28bdc0dd463e7a98e4dc',
    'SmallUpdateBlock': '1ac970d9e8125bddfcf6daa946e5a175077b3e008f73ddfd3dd06c7175249f79',
    'FlowHead': '1ba5bd4f558125144143db1b0dc78a8582ac259c76fb56360ceb73b4c38aefd0',
    'ConvGRU': 'b010df25f114ed0ff8e653c5b3a29627bfe1a094194b70234eaec607cff578ea',
    'SepConvGRU': 'b468244d28b547cf8886a66da5146e5c35b78ff8470db17775d9e266caa083df',
    'SmallMotionEncoder': 'aa75161b7b44c59c9452f986bc591bd17ab2898c4928b53115ec8717cce842e7',
    'BasicMotionEncoder': '5ea8b575090914b24dc7cc3a22327527324543d86de5cad66a4d627bd932b1b1',
}


@pytest.mark.parametrize('layer', sorted(SEEDED))
def test_seeded_default_weights_are_pinned(layer):
    from tf_raft_b200 import layers
    digest = hashlib.sha256()
    for seed in (0, 3):
        encoder = layer in ('BasicEncoder', 'SmallEncoder')
        for kwargs in [{'norm_type': nt} for nt in ('instance', 'batch', None)] if encoder else [{}]:
            for name, value in getattr(layers, layer)(device='cpu', seed=seed, **kwargs).params.items():
                digest.update(name.encode())
                digest.update(value.numpy().tobytes())
    assert digest.hexdigest() == SEEDED[layer]


@pytest.mark.gpu
def test_call_checks_status_and_runs_on_the_tensors_device():
    from tf_raft_b200 import _lib
    from tf_raft_b200.layers.corr import bilinear_sampler, upflow8
    out = torch.empty((1, 16, 16, 2), device='cuda')
    with pytest.raises(RuntimeError) as err:
        _lib.call('upflow8', out.device, _lib.ptr(None), 1, 2, 2, _lib.ptr(out))
    assert str(err.value) == 'raft_b200 upflow8 failed: [-1] bad argument (null pointer or unknown enum)'
    rng = np.random.default_rng(4)
    flow = rng.standard_normal((2, 6, 9, 2)).astype(np.float32)
    np.testing.assert_allclose(upflow8(torch.from_numpy(flow).cuda()).cpu().numpy(), corr_np.upflow8(flow),
                               atol=1e-5, rtol=1e-5)
    image = rng.standard_normal((8, 12, 10, 1)).astype(np.float32)
    coords = np.stack([rng.uniform(-2, 11, (8, 5, 5)), rng.uniform(-2, 13, (8, 5, 5))], axis=-1).astype(np.float32)
    got = bilinear_sampler(torch.from_numpy(image).cuda(), torch.from_numpy(coords).cuda()).cpu().numpy()
    np.testing.assert_array_equal(got, corr_np.bilinear_sampler(image, coords))


def test_every_binding_takes_as_many_arguments_as_the_header_declares():
    """ctypes calls with too few or too many arguments fail only when made; compare each signature with its declaration."""
    import re
    from tf_raft_b200 import _lib
    header = open(os.path.join(ROOT, 'include', 'raft_b200.h')).read()
    decls = {m.group(1): m.group(2).strip() for m in re.finditer(r'\b(raft_b200_\w+)\s*\(([^)]*)\)\s*;', header)}
    assert set(decls) == set(_lib._SIGNATURES)
    for name, params in decls.items():
        n = 0 if params in ('', 'void') else params.count(',') + 1
        assert len(_lib._SIGNATURES[name][1]) == n, f'{name}: {len(_lib._SIGNATURES[name][1])} bound, {n} declared'
