"""The stride-2 bf16 tensor-core entry points (pdae_conv_tc2_create_s2, pdae_conv_tc2_create_s2_dgrad,
pdae_wgrad_tc_create_bf16_s2, pdae_conv_s2_tc_supported) are declared, bound and validate their arguments before they touch
a device (no GPU needed)."""
import ctypes

import pytest

from pdae_b200 import _native

p = ctypes.c_void_p
CREATES = ("pdae_conv_tc2_create_s2", "pdae_conv_tc2_create_s2_dgrad", "pdae_wgrad_tc_create_bf16_s2")


def _create(fn, a, b, c, B=2, H=16, W=16, Cin=128, Cout=128, bias=None):
    L = _native.lib()
    h = ctypes.c_void_p()
    if fn == "pdae_conv_tc2_create_s2":
        rc = getattr(L, fn)(ctypes.byref(h), a, b, bias, c, B, H, W, Cin, Cout)
    else:
        rc = getattr(L, fn)(ctypes.byref(h), a, b, c, B, H, W, Cin, Cout)
    return rc, L.pdae_last_error()


def test_stride2_entry_points_are_bound():
    L = _native.lib()
    for fn in CREATES + ("pdae_conv_s2_tc_supported",):
        assert getattr(L, fn).restype == ctypes.c_int
    assert L.pdae_conv_tc2_create_s2_dgrad.argtypes == L.pdae_wgrad_tc_create_bf16_s2.argtypes
    assert len(L.pdae_conv_tc2_create_s2.argtypes) == len(L.pdae_conv_tc2_create_s2_dgrad.argtypes) + 1


def test_stride2_supported_predicate():
    L = _native.lib()
    for H, Cin, Cout in ((32, 64, 128), (16, 128, 128), (8, 128, 128), (64, 64, 128), (32, 128, 256), (16, 256, 256),
                         (8, 256, 256)):
        assert L.pdae_conv_s2_tc_supported(H, H, Cin, Cout) == 1
    assert L.pdae_conv_s2_tc_supported(64, 64, 3, 64) == 0       # the 3-channel stem stays on CUDA cores
    assert L.pdae_conv_s2_tc_supported(15, 16, 64, 64) == 0
    assert L.pdae_conv_s2_tc_supported(16, 16, 96, 64) == 0
    assert L.pdae_conv_s2_tc_supported(16, 16, 64, 32) == 0


@pytest.mark.parametrize("fn", CREATES)
def test_stride2_create_rejects_bad_arguments(fn):
    rc, msg = _create(fn, None, p(256), p(512))
    assert rc != 0 and b"null pointer" in msg
    rc, msg = _create(fn, p(256), None, p(512))
    assert rc != 0 and b"null pointer" in msg
    rc, msg = _create(fn, p(256), p(256), None)
    assert rc != 0 and b"null pointer" in msg
    rc, msg = _create(fn, p(264), p(256), p(512))
    assert rc != 0 and b"16-byte aligned" in msg
    rc, msg = _create(fn, p(256), p(256), p(512), H=15)
    assert rc != 0 and b"even" in msg
    rc, msg = _create(fn, p(256), p(256), p(512), W=9)
    assert rc != 0 and b"even" in msg
    rc, msg = _create(fn, p(256), p(256), p(512), Cin=96)
    assert rc != 0 and b"unsupported channels" in msg
    rc, msg = _create(fn, p(256), p(256), p(512), Cout=3)
    assert rc != 0 and b"unsupported channels" in msg


def test_stride2_forward_rejects_a_misaligned_bias():
    rc, msg = _create("pdae_conv_tc2_create_s2", p(256), p(256), p(512), bias=p(260))
    assert rc != 0 and b"16-byte aligned" in msg
