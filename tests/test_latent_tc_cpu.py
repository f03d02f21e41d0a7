"""The split-operand row kernels of the latent MLP's tensor-core sampling forward are exported, bound and recordable in a
native plan, and reject bad arguments before any CUDA call (no GPU needed)."""
import ctypes
import os

from pdae_b200 import _native

P = ctypes.c_void_p(16)      # an aligned dummy device pointer: validation fails before it is touched
f = ctypes.c_float


def _err(rc, text):
    assert rc != 0 and text in _native.lib().pdae_last_error(), _native.lib().pdae_last_error()


def test_split3_row_ops_exported_bound_and_recordable():
    L = _native.lib()
    table = open(os.path.join(os.path.dirname(_native.__file__), "csrc", "plan_exec_table.inc")).read()
    for name, sig in (("pdae_mlp_mod_ln_act_split3", "ppippfipiiiip"), ("pdae_copy_cols_split3", "ppiiiip")):
        assert hasattr(L, name) and name in _native.EXPORTS
        assert f'{{"{name}", (void*)&{name}, call_{sig}, {len(sig)}, "{sig}"}}' in table, name


def test_mlp_mod_ln_act_split3_validates_before_cuda():
    L = _native.lib()
    # cond rows narrower than N (cond_ld = 0, one shared row, is allowed)
    _err(L.pdae_mlp_mod_ln_act_split3(P, P, 100, None, None, f(1e-5), 1, P, 2560, 0, 4, 2048, None), b"bad args")
    # the written columns overrun a block of the split buffer
    _err(L.pdae_mlp_mod_ln_act_split3(P, P, 0, None, None, f(1e-5), 1, P, 2560, 1024, 4, 2048, None), b"bad args")
    _err(L.pdae_mlp_mod_ln_act_split3(P, None, 0, None, None, f(1e-5), 1, None, 512, 0, 4, 512, None), b"bad args")
    _err(L.pdae_mlp_mod_ln_act_split3(P, None, 0, None, None, f(1e-5), 1, P, 512, 0, 0, 512, None), b"bad args")
    _err(L.pdae_mlp_mod_ln_act_split3(P, None, 0, P, None, f(1e-5), 1, P, 512, 0, 4, 512, None), b"without bias")


def test_copy_cols_split3_validates_before_cuda():
    L = _native.lib()
    _err(L.pdae_copy_cols_split3(P, P, 2560, 2048, 4, 1024, None), b"bad args")
    _err(L.pdae_copy_cols_split3(P, P, 2560, -1, 4, 512, None), b"bad args")
    _err(L.pdae_copy_cols_split3(None, P, 512, 0, 4, 512, None), b"bad args")
    _err(L.pdae_copy_cols_split3(P, P, 512, 0, 0, 512, None), b"bad args")
