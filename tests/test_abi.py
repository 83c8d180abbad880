"""The C-ABI library loads, exports exactly what include/raft_b200.h declares, validates arguments
on the host, and the product package never touches the oracle.  No GPU needed."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))


@pytest.fixture(scope='module')
def L():
    from tf_raft_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_exports_match_header(L):
    from tf_raft_b200 import _lib
    header = open(os.path.join(ROOT, 'include', 'raft_b200.h')).read()
    declared = set(re.findall(r'\b(raft_b200_\w+)\s*\(', header))
    assert declared, 'no declarations parsed'
    assert declared == set(_lib.EXPORTED_SYMBOLS), declared ^ set(_lib.EXPORTED_SYMBOLS)
    for name in declared:
        assert hasattr(L, name), f'{name} not exported by libraft_b200.so'


def test_pyramid_sizes_match_survey(L):
    """SURVEY.md section 8(a) row a2: config 2 pyramid = 205.5 + 51.4 + 12.8 + 3.2 MB."""
    sizes = (ctypes.c_size_t * 4)()
    assert L.raft_b200_corr_pyramid_sizes(4, 56, 64, 4, sizes) == 0
    n = 4 * 56 * 64
    assert list(sizes) == [n * 56 * 64 * 4, n * 28 * 32 * 4, n * 14 * 16 * 4, n * 7 * 8 * 4]
    assert sum(sizes) == 272957440 + 0 or abs(sum(sizes) / 1e6 - 272.96) < 0.01


def test_host_side_argument_errors_and_abi_version(L):
    """ABI version 2: raft_b200_debug_timeline was removed from the header."""
    from tf_raft_b200 import _lib
    sizes = (ctypes.c_size_t * 8)()
    assert L.raft_b200_corr_pyramid_sizes(1, 8, 8, 0, sizes) == -1          # levels out of range
    assert L.raft_b200_corr_pyramid_sizes(1, 0, 8, 4, sizes) == -2          # bad dims
    assert L.raft_b200_corr_pyramid_sizes(1, 4, 4, 4, sizes) == -2          # level 3 would be empty
    assert L.raft_b200_corr_pyramid_sizes(1, 8, 8, 4, None) == -1
    nbytes = ctypes.c_size_t()
    assert L.raft_b200_update_workspace_bytes(0, 4, 56, 64, 1, ctypes.byref(nbytes)) == 0 and nbytes.value > 0
    assert L.raft_b200_update_workspace_bytes(7, 4, 56, 64, 1, ctypes.byref(nbytes)) == -1
    assert L.raft_b200_update_prepared_bytes(0, 324, 1, ctypes.byref(nbytes)) == 0 and nbytes.value > 12_000_000
    assert L.raft_b200_update_prepared_bytes(0, 196, 1, ctypes.byref(nbytes)) == -2
    assert L.raft_b200_update_prepared_bytes(1, 196, 0, ctypes.byref(nbytes)) == 0
    assert 'shape' in _lib.strerror(-2) and _lib.strerror(0) == 'ok'
    assert L.raft_b200_abi_version() == 2


def test_no_device_is_reported_not_emulated(L):
    if torch.cuda.is_available():
        pytest.skip('a GPU is present')
    assert L.raft_b200_device_ok(0) == -4


def test_cpu_tensors_are_rejected():
    """There is no CPU fallback: ops raise on CPU tensors instead of computing somewhere else."""
    import tf_raft_b200 as T
    f = torch.zeros(1, 8, 8, 64)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        T.CorrBlock(f, f)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        T.bilinear_sampler(torch.zeros(1, 4, 4, 1), torch.zeros(1, 3, 3, 2))
    with pytest.raises(NotImplementedError):
        T.tfa_sampler(torch.zeros(1, 4, 4, 1), torch.zeros(1, 3, 3, 2), mask=True)


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, 'tf_raft_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh', '.h')):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle', text, re.M), os.path.join(dirpath, f)


def test_losses_match_reference_known_answers():
    """reference tests/losses/test_losses.py:27-67 against the product's torch losses."""
    import numpy as np
    from tf_raft_b200 import end_point_error, sequence_loss
    flow_gt = np.array([[[0, 1], [0, 2], [0, 3]], [[0, 4], [0, 5], [0, 6]], [[0, 7], [0, 8], [0, 9]]]) - 0.1
    valid = np.array([[True, True, True], [True, True, True], [True, True, False]])
    flow_gt, valid = flow_gt[None].astype(np.float32), valid[None]
    preds = [np.zeros_like(flow_gt) for _ in range(6)]
    expect = sum(0.8 ** (5 - i) * np.mean(valid[..., None] * np.abs(p - flow_gt)) for i, p in enumerate(preds))
    np.testing.assert_almost_equal(float(sequence_loss((flow_gt, valid), preds)), expect, decimal=5)
    info = end_point_error([flow_gt, valid], preds[-1])
    np.testing.assert_almost_equal(float(info['epe']), np.mean(np.arange(1, 9) - 0.1), decimal=2)
    np.testing.assert_almost_equal(float(info['u3']), 3 / 8, decimal=2)


def test_workspace_and_shape_errors_are_detected_on_the_host(L):
    """Every entry point validates sizes before it launches anything: too-small workspaces / prepared buffers and
    inconsistent shapes come back as raft_status codes even without a GPU (pointers are never dereferenced here)."""
    fake = ctypes.c_void_p(0x1000)
    ptrs4 = (ctypes.c_void_p * 4)(0x1000, 0x2000, 0x3000, 0x4000)
    # correlation: F16X2 needs scratch
    assert L.raft_b200_corr_pyramid_build(fake, fake, 1, 8, 8, 64, 4, ptrs4, fake, 16, 1, None) == -3
    assert L.raft_b200_corr_pyramid_build(fake, fake, 1, 8, 8, 64, 4, ptrs4, None, 0, 1, None) == -3
    assert L.raft_b200_corr_pyramid_build(fake, fake, 1, 4, 8, 64, 4, ptrs4, fake, 1 << 30, 1, None) == -2   # level 3 empty
    assert L.raft_b200_corr_pyramid_build(None, fake, 1, 8, 8, 64, 4, ptrs4, fake, 1 << 30, 1, None) == -1
    # lookup: output row must hold levels*(2r+1)^2 channels
    assert L.raft_b200_corr_lookup(ptrs4, fake, 1, 8, 8, 4, 4, fake, 100, None) == -2
    # update block: workspace too small
    assert L.raft_b200_update_basic(fake, fake, fake, fake, fake, fake, fake, fake, 1, 8, 8, fake, 1024, 1, None) == -3
    assert L.raft_b200_update_small(fake, fake, fake, fake, fake, fake, fake, 1, 8, 8, fake, 1024, 0, None) == -3
    assert L.raft_b200_update_basic(fake, fake, fake, fake, fake, fake, None, fake, 1, 8, 8, fake, 1 << 40, 7, None) == -1   # bad precision
    # loop: radius / levels must match the variant's correlation channel count
    pyr = (ctypes.c_void_p * 4)(0x1000, 0x2000, 0x3000, 0x4000)
    ups = (ctypes.c_void_p * 2)(0x1000, 0x2000)
    assert L.raft_b200_forward_loop(0, fake, pyr, 4, 3, fake, fake, fake, ups, 2, 1, 8, 8, fake, 1 << 40, 1, None) == -2
    assert L.raft_b200_forward_loop(0, fake, pyr, 4, 4, fake, fake, fake, ups, 2, 1, 8, 8, fake, 64, 1, None) == -3
    # encoder
    nbytes = ctypes.c_size_t()
    assert L.raft_b200_encoder_prepared_bytes(0, 250, ctypes.byref(nbytes)) == -2        # out_dim must be a multiple of 32
    assert L.raft_b200_encoder_workspace_bytes(0, 4, 448, 512, ctypes.byref(nbytes)) == 0 and nbytes.value > (1 << 28)
    assert L.raft_b200_encoder_forward(0, 1, 256, fake, fake, 1, 64, 64, 0, 1, fake, fake, 1024, None) == -3
    assert L.raft_b200_conv2d(fake, fake, fake, 1, 8, 8, 4, 2, 3, 8, 0, fake, 8, 0, None) == -2      # even kernel size
