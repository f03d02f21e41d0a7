"""The entry points of the semantic encoder's tensor-core forward (pdae_conv_tc2_create_s2_ex, pdae_stem_conv_s2_bf16) are
declared, bound and check their arguments before they touch a device (no GPU needed)."""
import ctypes

import pytest

from pdae_b200 import _native
from pdae_b200._native import PDAE_BF16, PDAE_F32

p = ctypes.c_void_p


def _s2_ex(a=p(256), b=p(256), bias=None, out=p(512), odt=PDAE_BF16, stats=None, B=2, H=16, W=16, Cin=128, Cout=128):
    L = _native.lib()
    h = ctypes.c_void_p()
    rc = L.pdae_conv_tc2_create_s2_ex(ctypes.byref(h), a, b, bias, out, odt, stats, B, H, W, Cin, Cout)
    return rc, L.pdae_last_error()


def _stem(x=p(256), w=p(256), bias=None, out=p(512), stats=None, B=2, H=64, W=64, Cin=3, Cout=64):
    L = _native.lib()
    rc = L.pdae_stem_conv_s2_bf16(x, w, bias, out, stats, B, H, W, Cin, Cout, None)
    return rc, L.pdae_last_error()


def test_encoder_entry_points_are_bound():
    L = _native.lib()
    for fn in ("pdae_conv_tc2_create_s2_ex", "pdae_stem_conv_s2_bf16"):
        assert getattr(L, fn).restype == ctypes.c_int
    # the stride-2 stem takes the stride-1 stem's arguments; the extended forward adds out_dtype and ch_stats
    assert L.pdae_stem_conv_s2_bf16.argtypes == L.pdae_stem_conv_bf16.argtypes
    assert len(L.pdae_conv_tc2_create_s2_ex.argtypes) == len(L.pdae_conv_tc2_create_s2.argtypes) + 2


def test_stride2_ex_rejects_bad_arguments():
    for kw in (dict(a=None), dict(b=None), dict(out=None)):
        rc, msg = _s2_ex(**kw)
        assert rc != 0 and b"null pointer" in msg, kw
    L = _native.lib()
    rc = L.pdae_conv_tc2_create_s2_ex(None, p(256), p(256), None, p(512), PDAE_F32, None, 2, 16, 16, 128, 128)
    assert rc != 0 and b"null pointer" in L.pdae_last_error()
    for kw in (dict(a=p(264)), dict(b=p(260)), dict(out=p(520)), dict(bias=p(260))):
        rc, msg = _s2_ex(**kw)
        assert rc != 0 and b"16-byte aligned" in msg, kw
    rc, msg = _s2_ex(stats=p(1028))
    assert rc != 0 and b"8-byte aligned" in msg
    for kw in (dict(H=15), dict(W=9), dict(H=0), dict(B=0)):
        rc, msg = _s2_ex(**kw)
        assert rc != 0 and b"even" in msg, kw
    for kw in (dict(Cin=96), dict(Cout=3), dict(Cin=3)):
        rc, msg = _s2_ex(**kw)
        assert rc != 0 and b"unsupported channels" in msg, kw
    for odt in (2, -1, 7):
        rc, msg = _s2_ex(odt=odt)
        assert rc != 0 and b"out_dtype" in msg, odt


def test_stride2_forward_keeps_its_checks():
    """pdae_conv_tc2_create_s2 forwards to the extended entry point with an fp32 output and no statistics."""
    L = _native.lib()
    h = ctypes.c_void_p()
    rc = L.pdae_conv_tc2_create_s2(ctypes.byref(h), p(256), p(256), None, p(512), 2, 15, 16, 128, 128)
    assert rc != 0 and b"even" in L.pdae_last_error()


@pytest.mark.parametrize("kw,what", [
    (dict(x=None), b"null pointer"), (dict(w=None), b"null pointer"), (dict(out=None), b"null pointer"),
    (dict(x=p(260)), b"16-byte aligned"), (dict(out=p(520)), b"16-byte aligned"), (dict(stats=p(1026)), b"4-byte aligned"),
    (dict(H=63), b"even"), (dict(W=60), b"multiple of 8"), (dict(W=4), b"multiple of 8"), (dict(H=0), b"even"),
    (dict(Cin=0), b"image channels"), (dict(Cin=5), b"image channels"),
    (dict(Cout=60), b"multiple of 8"), (dict(Cout=512), b"multiple of 8"),
    (dict(B=0), b"B="), (dict(B=70000), b"B="),
])
def test_stride2_stem_rejects_bad_arguments(kw, what):
    rc, msg = _stem(**kw)
    assert rc != 0 and what in msg, (kw, msg)
