"""Build + ctypes binding of libpdae_b200.so (the C-ABI in include/pdae_b200.h).

The library is built in-tree by ``build()`` (called from ``__graft_entry__.build()``) with
``nvcc -gencode arch=compute_90a,code=sm_90a`` (Hopper, H100).  There is no CPU fallback anywhere in
this package: if the library is missing or the device is not sm_90, every compute path raises.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from ctypes import POINTER, c_char_p, c_float, c_int, c_int64, c_void_p
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
LIB_PATH = os.path.join(_HERE, "libpdae_b200.so")
SOURCES = ["conv_simt.cu", "norm_elementwise.cu", "attention_simt.cu", "conv_tc2.cu", "conv_tc3.cu", "wgrad_tc.cu", "plan_exec.cu", "backward_simt.cu", "train_io.cu"]

PDAE_F32, PDAE_BF16 = 0, 1
RESAMPLE_NONE, RESAMPLE_UP2, RESAMPLE_DOWN2 = 0, 1, 2

_lib: Optional[ctypes.CDLL] = None


class NativeError(RuntimeError):
    pass


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a into pdae_b200/libpdae_b200.so (cross-compiles without a GPU)."""
    srcs = [os.path.join(_HERE, "csrc", s) for s in SOURCES]
    deps = srcs + [os.path.join(_HERE, "csrc", "common.cuh"), os.path.join(_HERE, "csrc", "wgmma.cuh"),
                   os.path.join(_HERE, "csrc", "plan_exec_table.inc"),
                   os.path.join(_ROOT, "include", "pdae_b200.h")]
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(d) for d in deps):
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
           "-I", os.path.join(_ROOT, "include"), "-I", os.path.join(_HERE, "csrc"),
           "-shared", "-Xcompiler", "-fPIC", "-o", LIB_PATH] + srcs
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise NativeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return LIB_PATH


_P = c_void_p
_SIGS = {
    "pdae_last_error": (c_char_p, []),
    "pdae_abi_version": (c_int, []),
    "pdae_device_check": (c_int, []),
    "pdae_conv2d_simt": (c_int, [_P, c_int, c_int, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                 c_int, c_int, _P]),
    "pdae_conv3x3_smalln": (c_int, [_P, c_int, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "pdae_gn_stats": (c_int, [_P, c_int, _P, c_int, c_int, c_int, _P, _P]),
    "pdae_gn_coef": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_float, _P, c_int, _P, c_int, _P, _P]),
    "pdae_gn_apply": (c_int, [_P, c_int, c_int, _P, c_int, c_int, _P, c_int, c_int, c_int, c_int, c_int, _P, c_int, _P, c_int,
                              _P]),
    "pdae_zero": (c_int, [_P, c_int64, _P]),
    "pdae_ch_stats": (c_int, [_P, c_int, c_int, c_int, _P, _P]),
    "pdae_stats_det_workspace_bytes": (c_int64, [c_int, c_int, c_int]),
    "pdae_ch_stats_det": (c_int, [_P, c_int, c_int, c_int, _P, _P, c_int64, _P]),
    "pdae_gn_stats_det": (c_int, [_P, c_int, _P, c_int, c_int, c_int, _P, _P, c_int64, _P]),
    "pdae_gn_coef_ch": (c_int, [_P, c_int, _P, c_int, _P, _P, c_int, c_int, c_float, _P, c_int, _P, c_int, _P, _P]),
    "pdae_attention_simt": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "pdae_timestep_embedding": (c_int, [_P, c_int, c_int, _P, _P, _P]),
    "pdae_embedding_add": (c_int, [_P, _P, _P, c_int, c_int, _P]),
    "pdae_ddim_step": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int64, _P]),
    "pdae_ddim_select_t": (c_int, [_P, c_int, _P, c_int, _P, _P, c_int, _P]),
    "pdae_q_sample": (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int64, _P]),
    "pdae_noise_p_sample": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int64, _P]),
    "pdae_noise_p_sample_shift": (c_int, [_P, _P, _P, _P, _P, _P, c_int64, _P, _P, _P, _P, _P, _P, c_int, c_int64, _P]),
    "pdae_grad_blend": (c_int, [_P, _P, _P, _P, c_int64, _P]),
    "pdae_gap_terms_workspace_bytes": (c_int64, [c_int64]),
    "pdae_gap_terms": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int64, _P, c_int, c_int64, _P]),
    "pdae_mlp_mod_ln_act": (c_int, [_P, _P, _P, _P, c_float, c_int, _P, c_int, c_int, c_int, _P]),
    "pdae_copy_cols": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "pdae_mlp_mod_ln_act_bf16": (c_int, [_P, _P, c_int, _P, _P, c_float, c_int, _P, c_float, _P, c_int, c_int, c_int, _P]),
    "pdae_copy_cols_bf16": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "pdae_mlp_mod_ln_act_split3": (c_int, [_P, _P, c_int, _P, _P, c_float, c_int, _P, c_int, c_int, c_int, c_int, _P]),
    "pdae_copy_cols_split3": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "pdae_conv2d_dgrad_simt": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "pdae_conv2d_wgrad_simt": (c_int, [_P, c_int, c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "pdae_colsum": (c_int, [_P, c_int64, c_int, _P, _P]),
    "pdae_gn_bwd_sums": (c_int, [_P, c_int, _P, c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P]),
    "pdae_gn_bwd_coef": (c_int, [_P, _P, _P, _P, _P, c_int, _P, c_int, c_int, c_int, c_int, c_float, _P, _P, _P, _P, c_int, _P,
                                 c_int, _P]),
    "pdae_gn_bwd_apply": (c_int, [_P, c_int, _P, c_int, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, c_int, _P, _P, _P]),
    "pdae_embedding_bwd": (c_int, [_P, _P, _P, c_int, c_int, _P]),
    "pdae_conv2d_wgrad_simt_det_workspace_bytes": (c_int64, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "pdae_conv2d_wgrad_simt_det": (c_int, [_P, c_int, c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P,
                                           c_int64, _P]),
    "pdae_conv2d_dgrad_simt_det_workspace_bytes": (c_int64, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "pdae_conv2d_dgrad_simt_det": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, c_int64,
                                           _P]),
    "pdae_colsum_det_workspace_bytes": (c_int64, [c_int64, c_int]),
    "pdae_colsum_det": (c_int, [_P, c_int64, c_int, _P, _P, c_int64, _P]),
    "pdae_gn_bwd_sums_det_workspace_bytes": (c_int64, [c_int, c_int, c_int, c_int]),
    "pdae_gn_bwd_sums_det": (c_int, [_P, c_int, _P, c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, c_int64, _P]),
    "pdae_gn_bwd_coef_det_workspace_bytes": (c_int64, [c_int, c_int]),
    "pdae_gn_bwd_coef_det": (c_int, [_P, _P, _P, _P, _P, c_int, _P, c_int, c_int, c_int, c_int, c_float, _P, _P, _P, _P, c_int, _P,
                                     c_int, _P, c_int64, _P]),
    "pdae_embedding_bwd_det": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P]),
    "pdae_softmax_bwd": (c_int, [_P, _P, c_int64, c_int, c_float, _P]),
    "pdae_dsilu_mul": (c_int, [_P, _P, _P, c_int64, _P]),
    "pdae_add_inplace": (c_int, [_P, _P, c_int64, _P]),
    "pdae_mul_mask": (c_int, [_P, _P, c_float, c_int64, _P]),
    "pdae_nchw_to_nhwc": (c_int, [_P, _P, c_int, c_int, c_int, _P]),
    "pdae_gemm_batched_simt": (c_int, [_P, c_int64, c_int64, c_int64, c_int, _P, c_int64, c_int64, c_int64, c_int, _P, c_int64,
                                       c_int64, c_int64, c_int, c_int, c_int, c_int, c_int, c_float, _P]),
    "pdae_conv_tc2_create": (c_int, [POINTER(c_void_p), _P, _P, _P, _P, _P, c_int, _P, c_int, c_int, c_int, c_int, c_int, c_int,
                                     c_int, c_int]),
    "pdae_conv_tc2_create_skip": (c_int, [POINTER(c_void_p), _P, _P, _P, _P, _P, c_int, _P, c_int, _P, c_int, c_int, c_int, c_int,
                                          c_int, c_int, c_int]),
    "pdae_conv_tc2_create_skip2": (c_int, [POINTER(c_void_p), _P, _P, _P, _P, c_int, _P, c_int, _P, _P, c_int, _P, c_int, c_int,
                                           c_int, c_int, c_int, c_int, c_int]),
    "pdae_gemm_tc2_create": (c_int, [POINTER(c_void_p), _P, c_int64, c_int64, _P, c_int64, c_int64, _P, c_int, c_int64, c_int64,
                                     c_int, c_int, c_int, c_int]),
    "pdae_gemm_tc2_softmax_create": (c_int, [POINTER(c_void_p), _P, c_int64, c_int64, _P, c_int64, c_int64, _P, c_int64, c_int64,
                                             c_int, c_int, c_int, c_int, c_float]),
    "pdae_gemm_tc2_create_major": (c_int, [POINTER(c_void_p), _P, c_int, c_int64, c_int64, _P, c_int, c_int64, c_int64, _P,
                                           c_int64, c_int64, c_int, c_int, c_int, c_int]),
    "pdae_gemm_tc2_softmax_grad_create": (c_int, [POINTER(c_void_p), _P, c_int64, c_int64, _P, c_int64, c_int64, _P, c_int64,
                                                  c_int64, _P, c_int64, c_int64, c_int, c_int, c_int, c_int, c_float]),
    "pdae_conv_s2_tc_supported": (c_int, [c_int, c_int, c_int, c_int]),
    "pdae_conv_tc2_create_s2": (c_int, [POINTER(c_void_p), _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int]),
    "pdae_conv_tc2_create_s2_dgrad": (c_int, [POINTER(c_void_p), _P, _P, _P, c_int, c_int, c_int, c_int, c_int]),
    "pdae_conv_tc2_create_s2_ex": (c_int, [POINTER(c_void_p), _P, _P, _P, _P, c_int, _P, c_int, c_int, c_int, c_int, c_int]),
    "pdae_conv_tc2_create_splitk": (c_int, [POINTER(c_void_p), _P, _P, _P, _P, c_int, c_int, c_int]),
    "pdae_conv_tc2_run": (c_int, [_P, _P]),
    "pdae_conv_tc2_det_workspace_bytes": (c_int64, [_P]),
    "pdae_conv_tc2_set_deterministic": (c_int, [_P, _P, c_int64]),
    "pdae_conv_tc2_set_head_fuse": (c_int, [_P, _P]),
    "pdae_conv_tc3_supported": (c_int, [c_int, c_int, c_int, c_int]),
    "pdae_conv_tc3_create": (c_int, [POINTER(c_void_p), _P, c_int, _P, c_int, c_int, _P, c_int, _P, _P, _P, c_int, _P, c_int, _P, _P,
                                     _P, c_int, _P, c_int, c_int, c_int, c_int, c_int]),
    "pdae_conv_tc3_run": (c_int, [_P, _P]),
    "pdae_conv_tc3_det_workspace_bytes": (c_int64, [_P]),
    "pdae_conv_tc3_set_deterministic": (c_int, [_P, _P, c_int64]),
    "pdae_conv_tc3_destroy": (None, [_P]),
    "pdae_wgrad_tc_supported": (c_int, [c_int, c_int, c_int, c_int, c_int]),
    "pdae_wgrad_tc_create": (c_int, [POINTER(c_void_p), _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int]),
    "pdae_wgrad_tc_create_bf16": (c_int, [POINTER(c_void_p), _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int]),
    "pdae_wgrad_tc_create_bf16_s2": (c_int, [POINTER(c_void_p), _P, _P, _P, c_int, c_int, c_int, c_int, c_int]),
    "pdae_wgrad_tc_det_workspace_bytes": (c_int64, [_P]),
    "pdae_wgrad_tc_set_deterministic": (c_int, [_P, _P, c_int64]),
    "pdae_wgrad_tc_run": (c_int, [_P, _P]),
    "pdae_wgrad_tc_destroy": (None, [_P]),
    "pdae_softmax_bf16": (c_int, [_P, _P, c_int64, c_int, c_float, _P]),
    "pdae_transpose_v": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "pdae_qkv_split3": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "pdae_softmax_split3": (c_int, [_P, _P, c_int64, c_int, c_float, _P]),
    "pdae_conv_tc2_destroy": (None, [_P]),
    "pdae_mlp_mod_ln_act_bwd": (c_int, [_P, _P, _P, _P, c_float, c_int, _P, c_int, _P, _P, _P, _P, c_int, c_int, _P]),
    "pdae_mlp_mod_ln_act_bwd_bf16": (c_int, [_P, _P, c_int, _P, _P, c_float, c_int, _P, c_int, _P, c_float, _P, _P, _P, _P, _P, _P,
                                             c_int, c_int, _P]),
    "pdae_mul_mask_cols": (c_int, [_P, c_int, _P, c_float, c_int, c_int, _P]),
    "pdae_stem_conv_bf16": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "pdae_stem_conv_s2_bf16": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "pdae_stem_conv_det_workspace_bytes": (c_int64, [c_int, c_int, c_int, c_int, c_int]),
    "pdae_stem_conv_bf16_det": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P]),
    "pdae_gn_apply_split3": (c_int, [_P, c_int, _P, c_int, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, c_int, _P]),
    "pdae_adam_ema_step": (c_int, [_P, _P, c_int, c_int, c_float, c_float, c_float, c_float, c_float, c_int64, c_float,
                                   c_float, _P]),
    "pdae_unpack_grads": (c_int, [_P, _P, c_int, c_int, _P, _P]),
    "pdae_plan_create": (c_int, [POINTER(c_void_p)]),
    "pdae_plan_add": (c_int, [_P, c_char_p, _P, c_int, c_int]),
    "pdae_plan_run_step": (c_int, [_P, _P]),
    "pdae_plan_size": (c_int, [_P]),
    "pdae_plan_op_name": (c_char_p, [_P, c_int]),
    "pdae_plan_destroy": (None, [_P]),
    "pdae_images_to_u8_nhwc": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "pdae_u8_nhwc_to_images": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "pdae_mse_per_image": (c_int, [_P, _P, c_int, c_int64, _P, _P, _P]),
    "pdae_ssim_per_image": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P, _P, _P]),
    "pdae_mse_det_workspace_bytes": (c_int64, [c_int, c_int64]),
    "pdae_mse_per_image_det": (c_int, [_P, _P, c_int, c_int64, _P, c_int64, _P, _P]),
    "pdae_ssim_det_workspace_bytes": (c_int64, [c_int, c_int, c_int, c_int]),
    "pdae_ssim_per_image_det": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P, c_int64, _P, _P]),
}
EXPORTS = tuple(_SIGS.keys())


def lib() -> ctypes.CDLL:
    """Load the native library (never builds implicitly; never falls back)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeError(f"{LIB_PATH} is missing -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(pdae_b200 has no CPU fallback)")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def pack_args(cfn, cargs) -> bytes:
    """Argument values of one recorded call as an array of `pdae_arg` (8-byte union: pointer / int64 / double), in the entry
    point's declared order; a None (stream placeholder, null pointer) becomes 0."""
    import struct
    out = []
    assert len(cargs) == len(cfn.argtypes), (cfn.__name__, len(cargs), len(cfn.argtypes))
    for t, a in zip(cfn.argtypes, cargs):
        v = a.value if isinstance(a, ctypes._SimpleCData) else a
        if t is c_float:
            out.append(struct.pack("<d", float(v)))
        elif t is c_void_p:
            out.append(struct.pack("<Q", int(v) if v else 0))
        elif t in (c_int, c_int64):
            out.append(struct.pack("<q", int(v)))
        else:
            raise NativeError(f"{cfn.__name__}: argument type {t} cannot be recorded in a native plan")
    return b"".join(out)


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().pdae_last_error()
        raise NativeError(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")


def require_device() -> None:
    check(lib().pdae_device_check(), "pdae_device_check")
