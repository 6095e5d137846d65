"""CPU: the native BatchNorm's channel limits -- the block tails (forms 1, 2) up to 2048 channels, Resnet50_8s's
layer4 bn3 and its downsample's BatchNorm; act(bn(x)) (form 0) still up to 1024 -- checked without a GPU."""
import ctypes

import pytest

from pvnet_b200 import _native


@pytest.mark.parametrize("form", [1, 2])
def test_block_tails_take_2048_channels(form):
    L = _native.lib()
    n = ctypes.c_size_t()
    assert L.pvnet_batchnorm_workspace_bytes(form, 2048, 1000, ctypes.byref(n)) == 0
    assert n.value >= (4 if form == 2 else 2) * 2048 * 4 * 8
    assert L.pvnet_batchnorm_workspace_bytes(form, 1536, 1000, ctypes.byref(n)) == 0
    assert L.pvnet_batchnorm_workspace_bytes(form, 2052, 1000, ctypes.byref(n)) == -1
    assert b"2048" in L.pvnet_last_error()


def test_form0_keeps_its_1024_channel_limit():
    L = _native.lib()
    n = ctypes.c_size_t()
    assert L.pvnet_batchnorm_workspace_bytes(0, 1024, 1000, ctypes.byref(n)) == 0
    assert L.pvnet_batchnorm_workspace_bytes(0, 1028, 1000, ctypes.byref(n)) == -1
    p = _native.BatchNormParams(None, None, None, None, 1, 0.1, 1e-5, 256, 256)
    fake = ctypes.c_void_p(1 << 20)
    # the forward refuses a 2048-channel form 0 before it touches a pointer; a form 1 call of that width passes the
    # channel check and stops at the workspace check
    assert L.pvnet_batchnorm_act_forward(0, 1, fake, None, 100, 2048, ctypes.byref(p), None, fake, fake, 1 << 30,
                                         None) == -1
    assert b"up to 1024" in L.pvnet_last_error()
    assert L.pvnet_batchnorm_act_forward(1, 1, fake, fake, 100, 2048, ctypes.byref(p), None, fake, fake, 16,
                                         None) == -1
    assert b"workspace" in L.pvnet_last_error()
