"""The attention-backward tensor-core entry points (pdae_gemm_tc2_create_major, pdae_gemm_tc2_softmax_grad_create) are declared,
bound and validate their arguments before they touch a device (no GPU needed)."""
import ctypes

import pytest

from pdae_b200 import _native

p = ctypes.c_void_p


def _major(a=p(256), b=p(512), out=p(1024), a_mn=1, b_mn=1, lds=(256, 256 * 256, 192, 256 * 192, 192, 256 * 192),
           batch=2, M=256, N=64, K=256):
    L = _native.lib()
    h = ctypes.c_void_p()
    a_ld, a_bs, b_ld, b_bs, o_ld, o_bs = lds
    rc = L.pdae_gemm_tc2_create_major(ctypes.byref(h), a, a_mn, a_ld, a_bs, b, b_mn, b_ld, b_bs, out, o_ld, o_bs, batch, M, N, K)
    return rc, L.pdae_last_error()


def _sgrad(a=p(256), b=p(512), pr=p(768), out=p(1024), lds=(64, 256 * 64, 192, 256 * 192, 256, 256 * 256, 256, 256 * 256),
           batch=2, M=256, N=256, K=64, alpha=0.125):
    L = _native.lib()
    h = ctypes.c_void_p()
    a_ld, a_bs, b_ld, b_bs, p_ld, p_bs, o_ld, o_bs = lds
    rc = L.pdae_gemm_tc2_softmax_grad_create(ctypes.byref(h), a, a_ld, a_bs, b, b_ld, b_bs, pr, p_ld, p_bs, out, o_ld, o_bs,
                                             batch, M, N, K, alpha)
    return rc, L.pdae_last_error()


def test_attention_backward_entry_points_are_bound():
    L = _native.lib()
    for fn in ("pdae_gemm_tc2_create_major", "pdae_gemm_tc2_softmax_grad_create"):
        assert getattr(L, fn).restype == ctypes.c_int
    assert len(L.pdae_gemm_tc2_create_major.argtypes) == 16
    assert len(L.pdae_gemm_tc2_softmax_grad_create.argtypes) == 18
    assert L.pdae_gemm_tc2_softmax_grad_create.argtypes[-1] is ctypes.c_float


def test_create_functions_are_not_recorded_by_the_plan_executor():
    # (they take a plan handle out-pointer; the executor replays pdae_conv_tc2_run on the handle they create)
    import importlib.util
    import os
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("gen_plan_exec", os.path.join(here, "scripts", "gen_plan_exec.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    names = [n for n, _ in gen.recordable()]
    assert "pdae_conv_tc2_run" in names
    assert "pdae_gemm_tc2_create_major" not in names and "pdae_gemm_tc2_softmax_grad_create" not in names


@pytest.mark.parametrize("a_mn,b_mn", [(1, 1), (0, 1), (1, 0)])
def test_major_gemm_rejects_bad_arguments(a_mn, b_mn):
    for kw in (dict(a=None), dict(b=None), dict(out=None)):
        rc, msg = _major(a_mn=a_mn, b_mn=b_mn, **kw)
        assert rc != 0 and b"null pointer" in msg
    for kw in (dict(a=p(264)), dict(b=p(520)), dict(out=p(1028))):
        rc, msg = _major(a_mn=a_mn, b_mn=b_mn, **kw)
        assert rc != 0 and b"16-byte aligned" in msg
    rc, msg = _major(a_mn=a_mn, b_mn=b_mn, lds=(260, 256 * 256, 192, 256 * 192, 192, 256 * 192))
    assert rc != 0 and b"multiples of 16 bytes" in msg
    rc, msg = _major(a_mn=a_mn, b_mn=b_mn, lds=(256, 256 * 256, 192, 256 * 192, 0, 256 * 192))
    assert rc != 0 and b"multiples of 16 bytes" in msg
    for kw in (dict(M=192), dict(N=96), dict(K=200), dict(batch=0), dict(M=0)):
        rc, msg = _major(a_mn=a_mn, b_mn=b_mn, **kw)
        assert rc != 0 and b"M % 128" in msg, kw


def test_major_gemm_rejects_bad_major_flags():
    for a_mn, b_mn in ((2, 0), (0, -1)):
        rc, msg = _major(a_mn=a_mn, b_mn=b_mn)
        assert rc != 0 and b"major flags" in msg


def test_softmax_grad_gemm_rejects_bad_arguments():
    for kw in (dict(a=None), dict(b=None), dict(pr=None), dict(out=None)):
        rc, msg = _sgrad(**kw)
        assert rc != 0 and b"null pointer" in msg, kw
    for kw in (dict(a=p(264)), dict(b=p(520)), dict(pr=p(776)), dict(out=p(1032))):
        rc, msg = _sgrad(**kw)
        assert rc != 0 and b"16-byte aligned" in msg, kw
    rc, msg = _sgrad(lds=(64, 256 * 64, 192, 256 * 192, 250, 256 * 256, 256, 256 * 256))
    assert rc != 0 and b"multiples of 16 bytes" in msg
    for kw in (dict(M=64), dict(K=32), dict(batch=-1)):
        rc, msg = _sgrad(**kw)
        assert rc != 0 and b"M % 128" in msg, kw
    rc, msg = _sgrad(N=192)
    assert rc != 0 and b"must be 64, 128 or 256" in msg
    rc, msg = _sgrad(N=512)
    assert rc != 0 and b"must be 64, 128 or 256" in msg
    for alpha in (0.0, -0.5):
        rc, msg = _sgrad(alpha=alpha)
        assert rc != 0 and b"alpha must be positive" in msg
