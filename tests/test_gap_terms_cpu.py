"""pdae_gap_terms and its workspace query (include/pdae_b200.h) on the host: the workspace size follows the element count, and
bad arguments fail with -1 and a message in pdae_last_error() before any CUDA call -- directly and through the C-ABI plan
executor -- so no GPU is needed."""
import ctypes

import pytest

from pdae_b200 import _native

P = ctypes.c_void_p(16)                  # never dereferenced: every call below fails its argument checks first


def _args(**kw):
    a = dict(x0=P, x_t=P, eps=P, grad=P, t=P, c0=P, c1=P, A=P, Bm=P, shift=P, ws=P, ws_bytes=1 << 20, out=P, B=2,
             per_sample=48, stream=None)
    a.update(kw)
    return list(a.values())


def test_workspace_bytes_follow_the_element_count():
    L = _native.lib()
    # two fp64 partials per block of 4096 elements
    assert L.pdae_gap_terms_workspace_bytes(1) == 16
    assert L.pdae_gap_terms_workspace_bytes(4096) == 16
    assert L.pdae_gap_terms_workspace_bytes(4097) == 32
    assert L.pdae_gap_terms_workspace_bytes(100 * 3 * 128 * 128) == 1200 * 16
    assert L.pdae_gap_terms_workspace_bytes(0) < 0 and b"must be > 0" in L.pdae_last_error()
    assert L.pdae_gap_terms_workspace_bytes(-5) < 0


@pytest.mark.parametrize("kw,msg", [
    (dict(x0=None), b"null pointer"),
    (dict(grad=None), b"null pointer"),
    (dict(t=None), b"null pointer"),
    (dict(shift=None), b"null pointer"),
    (dict(ws=None), b"null pointer"),
    (dict(out=None), b"null pointer"),
    (dict(B=0), b"B=0 and per_sample=48 must be > 0"),
    (dict(B=-3), b"B=-3"),
    (dict(per_sample=0), b"per_sample=0 must be > 0"),
    (dict(B=2, per_sample=4097, ws_bytes=16), b"workspace of 16 bytes, 48 needed"),
])
def test_bad_arguments_fail_before_the_device(kw, msg):
    L = _native.lib()
    assert L.pdae_gap_terms(*_args(**kw)) == -1
    assert msg in L.pdae_last_error(), L.pdae_last_error()


def _run_recorded(args):
    L = _native.lib()
    h = ctypes.c_void_p()
    _native.check(L.pdae_plan_create(ctypes.byref(h)), "pdae_plan_create")
    try:
        blob = _native.pack_args(L.pdae_gap_terms, args)
        _native.check(L.pdae_plan_add(h, b"pdae_gap_terms", blob, len(args), len(args) - 1), "pdae_plan_add")
        assert L.pdae_plan_run_step(h, None) == -1
        return L.pdae_last_error()
    finally:
        L.pdae_plan_destroy(h)


def test_recorded_in_a_native_plan():
    """The generated trampoline passes every argument in order: pointer, int and int64 values reach the entry point's checks."""
    assert b"B=0 and per_sample=12345 must be > 0" in _run_recorded(_args(B=0, per_sample=12345))
    assert b"workspace of 16 bytes, 48 needed" in _run_recorded(_args(per_sample=5000, ws_bytes=16))
    assert b"gap_terms: null pointer" in _run_recorded(_args(x0=None))
    # int64 values beyond 32 bits: 2^29 + 2 blocks need 2^33 + 32 bytes
    err = _run_recorded(_args(B=1, per_sample=(1 << 41) + 8192, ws_bytes=(1 << 33) + 16))
    assert b"workspace of 8589934608 bytes, 8589934624 needed" in err, err
