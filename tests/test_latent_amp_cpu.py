"""The latent-MLP autocast entry points are exported and bound, and reject bad arguments before any CUDA call (no GPU
needed)."""
import ctypes

from pdae_b200 import _native

P = ctypes.c_void_p(16)      # an aligned dummy device pointer: validation fails before it is touched


def _err(rc, text):
    assert rc != 0 and text in _native.lib().pdae_last_error(), _native.lib().pdae_last_error()


def test_splitk_create_validates_before_cuda():
    L = _native.lib()
    h = ctypes.c_void_p()
    _err(L.pdae_conv_tc2_create_splitk(ctypes.byref(h), P, P, None, P, 128, 512, 500), b"Cout % 64 == 0")
    _err(L.pdae_conv_tc2_create_splitk(ctypes.byref(h), P, P, None, P, 128, 500, 512), b"not a multiple of 64")
    _err(L.pdae_conv_tc2_create_splitk(ctypes.byref(h), P, P, None, P, 0, 512, 512), b"B=0")
    _err(L.pdae_conv_tc2_create_splitk(ctypes.byref(h), None, P, None, P, 128, 512, 512), b"null pointer")
    _err(L.pdae_conv_tc2_create_splitk(ctypes.byref(h), P, P, None, ctypes.c_void_p(20), 128, 512, 512), b"16-byte aligned")


def test_bf16_row_ops_validate_before_cuda():
    L = _native.lib()
    f = ctypes.c_float
    _err(L.pdae_mlp_mod_ln_act_bf16(P, P, 100, None, None, f(1e-5), 1, None, f(1.0), P, 256, 4, 256, None), b"bad args")
    _err(L.pdae_mlp_mod_ln_act_bf16(P, None, 0, P, None, f(1e-5), 1, None, f(1.0), P, 256, 4, 256, None), b"without bias")
    _err(L.pdae_copy_cols_bf16(P, P, 512, 256, 4, 512, None), b"bad args")
    _err(L.pdae_mlp_mod_ln_act_bwd_bf16(P, P, 256, None, None, f(1e-5), 1, P, 256, None, f(1.0), P, None, None, None, None,
                                        None, 4, 256, None), b"bad args")
    _err(L.pdae_mlp_mod_ln_act_bwd_bf16(P, None, 256, None, None, f(1e-5), 1, P, 256, None, f(1.0), P, P, P, P, None, None,
                                        4, 256, None), b"dcond without cond")
    _err(L.pdae_mlp_mod_ln_act_bwd_bf16(P, P, 100, None, None, f(1e-5), 1, P, 256, None, f(1.0), P, P, P, P, None, None,
                                        4, 256, None), b"cond_ld=100")
