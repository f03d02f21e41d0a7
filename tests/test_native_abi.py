"""The C-ABI library builds for sm_90a, loads, and exports every symbol include/pdae_b200.h declares (no GPU needed)."""
import ctypes
import os
import re

from pdae_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "pdae_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pdae_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported_and_bound():
    _native.build()
    lib = ctypes.CDLL(_native.LIB_PATH)
    syms = declared_symbols()
    assert len(syms) >= 18
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/pdae_b200.h but not exported"
    assert sorted(_native.EXPORTS) == syms, "ctypes bindings out of sync with the header"


def test_abi_version_and_error_string():
    L = _native.lib()
    assert L.pdae_abi_version() == 1
    # argument validation happens before any CUDA call, so it is testable without a device
    rc = L.pdae_conv3x3_smalln(None, 0, None, None, None, 1, 8, 8, 64, 3, None)
    assert rc == -1 and b"null pointer" in L.pdae_last_error()
    rc = L.pdae_gn_stats(ctypes.c_void_p(16), 30, None, 0, 1, 64, ctypes.c_void_p(16), None)
    assert rc == -1 and b"unsupported" in L.pdae_last_error()


def test_sass_is_hopper_native():
    """wgmma -> HGMMA, TMA load / store -> UTMALDG / UTMASTG must be present in the sm_90a cubin."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        import pytest
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _native.LIB_PATH], capture_output=True, text=True).stdout
    for mnem in ("HGMMA", "UTMALDG", "UTMASTG"):
        assert mnem in sass, mnem
    assert "sm_90a" in sass


def test_gn_bwd_down2_rejects_odd_dims_before_any_launch():
    """DOWN2 backward reads dy at (y/2, x/2) of an [H/2][W/2] tensor: an odd H or W would read past its end.  Both passes
    that gather dy refuse it, like the forward, before touching the stream (dummy pointers are never dereferenced)."""
    L = _native.lib()
    p = ctypes.c_void_p(16)
    for H, W in ((7, 8), (8, 9)):
        rc = L.pdae_gn_bwd_sums(p, 64, None, 0, p, p, 1, 2, 2, H, W, p, None)
        assert rc == -1 and b"odd dims for DOWN2" in L.pdae_last_error(), (H, W)
        rc = L.pdae_gn_bwd_apply(p, 64, None, 0, p, p, p, 1, 2, 2, H, W, None, 0, p, None, None)
        assert rc == -1 and b"odd dims for DOWN2" in L.pdae_last_error(), (H, W)


def test_qkv_split3_rejects_odd_T_before_any_launch():
    L = _native.lib()
    p = ctypes.c_void_p(16)
    rc = L.pdae_qkv_split3(p, p, p, p, 2, 63, 64, 2, 0, None)
    assert rc == -1 and b"T must be even" in L.pdae_last_error()
