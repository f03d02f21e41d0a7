"""The single-pass bf16 weight-gradient entry point (pdae_wgrad_tc_create_bf16) is declared, bound and validates its arguments
before it touches a device (no GPU needed)."""
import ctypes

from pdae_b200 import _native


def _create(act, dy, dw, B=2, H=16, W=16, Cin=128, Cout=128, k=3):
    L = _native.lib()
    h = ctypes.c_void_p()
    rc = L.pdae_wgrad_tc_create_bf16(ctypes.byref(h), act, dy, dw, B, H, W, Cin, Cout, k)
    return rc, L.pdae_last_error()


def test_wgrad_tc_create_bf16_is_bound_like_the_split_variant():
    L = _native.lib()
    assert L.pdae_wgrad_tc_create_bf16.argtypes == L.pdae_wgrad_tc_create.argtypes
    assert L.pdae_wgrad_tc_create_bf16.restype == L.pdae_wgrad_tc_create.restype


def test_wgrad_tc_create_bf16_rejects_bad_arguments():
    p = ctypes.c_void_p
    rc, msg = _create(None, p(256), p(512))
    assert rc != 0 and b"null pointer" in msg
    rc, msg = _create(p(256), p(256), p(512), Cin=96)
    assert rc != 0 and b"unsupported shape" in msg
    rc, msg = _create(p(256), p(256), p(512), k=5)
    assert rc != 0 and b"unsupported shape" in msg
    rc, msg = _create(p(264), p(256), p(512))
    assert rc != 0 and b"16-byte aligned" in msg
