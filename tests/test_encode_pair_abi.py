"""raft_b200_encode_pair validates its arguments on the host, before it forks or launches anything.  No GPU needed."""
import ctypes

import pytest


@pytest.fixture(scope='module')
def L():
    from tf_raft_b200 import build, _lib
    build.build()
    return _lib.lib()


def test_encode_pair_workspace_and_argument_errors(L):
    n = ctypes.c_size_t()
    enc = ctypes.c_size_t()
    assert L.raft_b200_encode_pair_workspace_bytes(0, 4, 448, 512, 256, ctypes.byref(n)) == 0
    assert L.raft_b200_encoder_workspace_bytes(0, 4, 448, 512, ctypes.byref(enc)) == 0
    assert n.value >= 3 * enc.value + 4 * 56 * 64 * 256 * 4            # three encoder workspaces and cnet's output
    assert L.raft_b200_encode_pair_workspace_bytes(5, 4, 448, 512, 256, ctypes.byref(n)) == -1
    assert L.raft_b200_encode_pair_workspace_bytes(0, 0, 448, 512, 256, ctypes.byref(n)) == -2

    fake = ctypes.c_void_p(0x1000)

    def call(variant=0, fnet_dim=256, hidden=128, context=128, H=64, W=64, ws_bytes=1 << 40, image1=fake):
        return L.raft_b200_encode_pair(variant, fake, 1, fnet_dim, fake, 2, hidden, context, image1, fake, 1, H, W, fake,
                                       fake, fake, fake, fake, ws_bytes, None)

    assert call(image1=None) == -1                                          # null pointer
    assert call(variant=3) == -1                                            # unknown variant
    assert call(fnet_dim=250) == -2                                         # out_dim must be a multiple of 32
    assert call(hidden=128, context=160) == -2                              # cnet's width above 256
    assert call(H=4) == -2                                                  # smaller than one feature cell
    assert call(ws_bytes=1024) == -3                                        # pair workspace too small
