"""Deterministic training without a GPU: the deterministic backward kernels contain no float atomic in their SASS (and the same
matcher finds the atomics of the default ones), their entry points refuse bad arguments and short workspaces before any
launch, and the trainer caches are keyed by torch.use_deterministic_algorithms."""
import ctypes
import re

import pytest
import torch

from pdae_b200 import _native
from pdae_b200.engine import DET_OPS, NONDET_OPS, det_entry_points
from tests.test_deterministic_cpu import _atomics, _functions

DET_BACKWARD_KERNELS = {
    # (mangled-name pattern, instances expected)
    r"wgrad_tc_kernelILi\d+ELb[01]ELb[01]ELb1EE": 6,          # DET = true: BN 64/128 x split / bf16 / stride-2
    r"conv_wgrad_kernelILb1EE": 1,
    r"colsum_kernelILb1EE": 1,
    r"colsum_v4_kernelILb1EE": 1,
    r"gn_bwd_sums_kernelILi\dELb1EE": 3,                      # every resample mode
    r"gn_bwd_coef_kernelILb1EE": 1,
    r"gn_param_reduce_kernel": 1,
    r"embedding_bwd_det_kernel": 1,
    r"linear_dgrad_splitk_kernelILb1EE": 1,
    r"slot_sum_kernel": 1,
    # conv_tc2 DET instantiations of the training GEMMs (GM_A_MN = 1, GM_B_MN = 2, both = 3, softmax gradient 4 / 12) and of
    # the stride-2 data gradient (S2 = 2)
    r"conv_tc2_kernelILi(64|128)ELb0ELi0ELi[123]ELb1EE": 6,
    r"conv_tc2_kernelILi(64|128)ELb1ELi0ELi(4|12)ELb1EE": 3,
    r"conv_tc2_kernelILi(64|128)ELb0ELi2ELi0ELb1EE": 2,
}
# the rest of the backward and the optimizer: atomic-free as they are (shown, not assumed)
ATOMIC_FREE = (r"conv_dgrad_kernel", r"conv3x3_dgrad_smalln_kernel", r"gemm_batched_kernel", r"softmax_bwd_kernel",
               r"gn_bwd_apply_kernel", r"unpack_grads_kernel", r"adam_ema_kernel")


def test_deterministic_backward_kernels_have_no_float_atomics():
    funcs = _functions()
    for pat, n in DET_BACKWARD_KERNELS.items():
        hits = [f for f in funcs if re.search(pat, f)]
        assert len(hits) >= n, (pat, hits)
        for f in hits:
            assert not _atomics(funcs[f]), (f, _atomics(funcs[f]))
    for pat in ATOMIC_FREE:
        hits = [f for f in funcs if re.search(pat, f)]
        assert hits, pat
        for f in hits:
            assert not _atomics(funcs[f]), (f, _atomics(funcs[f]))

    # the same matcher sees the atomics of the default kernels the deterministic ones replace
    def found(pat):
        return set().union(*[_atomics(b) for f, b in funcs.items() if re.search(pat, f)])
    for pat in (r"wgrad_tc_kernelILi128ELb1ELb0ELb0EE", r"conv_wgrad_kernelILb0EE", r"colsum_v4_kernelILb0EE",
                r"colsum_kernelILb0EE", r"gn_bwd_sums_kernelILi0ELb0EE", r"gn_bwd_coef_kernelILb0EE",
                r"linear_dgrad_splitk_kernelILb0EE", r"embedding_bwd_kernel", r"conv_tc2_kernelILi128ELb0ELi0ELi1ELb0EE",
                r"conv_tc2_kernelILi128ELb0ELi2ELi0ELb0EE"):
        assert "REDG.E.ADD.F32" in found(pat), pat
    assert "ATOMS.CAST.SPIN" in found(r"gn_bwd_sums_kernelILi0ELb0EE")


def _err(L):
    return L.pdae_last_error().decode()


def test_backward_entry_points_reject_bad_arguments_before_any_launch():
    """Dummy pointers are never dereferenced: every call below fails its argument checks."""
    L = _native.lib()
    p = ctypes.c_void_p(16)
    i64 = ctypes.c_int64
    # CUDA-core weight gradient: a 64-px encoder conv splits over pixel chunks, a one-pixel Linear bank does not
    n = L.pdae_conv2d_wgrad_simt_det_workspace_bytes(8, 64, 64, 3, 64, 3, 2, 1)
    assert n > 0 and n % (27 * 64 * 4) == 0
    assert L.pdae_conv2d_wgrad_simt_det_workspace_bytes(8, 1, 1, 512, 4096, 1, 1, 0) == 0
    assert L.pdae_conv2d_wgrad_simt_det_workspace_bytes(0, 64, 64, 3, 64, 3, 2, 1) < 0
    assert L.pdae_conv2d_wgrad_simt_det(p, 1, 0, p, p, 8, 64, 64, 3, 64, 3, 2, 1, p, i64(n - 4), None) == -1
    assert "workspace" in _err(L)
    assert L.pdae_conv2d_wgrad_simt_det(p, 1, 0, p, p, 8, 64, 64, 3, 64, 3, 2, 1, None, i64(n), None) == -1
    assert L.pdae_conv2d_wgrad_simt_det(None, 1, 0, p, p, 8, 64, 64, 3, 64, 3, 2, 1, p, i64(n), None) == -1
    # data gradient: only the wide-Linear split-K form needs slots, one per 64 output rows
    assert L.pdae_conv2d_dgrad_simt_det_workspace_bytes(4, 1, 1, 512, 4096, 1, 1, 0, 0) == 64 * 4 * 512 * 4
    assert L.pdae_conv2d_dgrad_simt_det_workspace_bytes(4, 16, 16, 64, 64, 3, 1, 1, 0) == 0
    assert L.pdae_conv2d_dgrad_simt_det(p, p, p, 4, 1, 1, 512, 4096, 1, 1, 0, 0, p, i64(1024), None) == -1
    assert "workspace" in _err(L)
    # bias gradient: row chunks of pdae_colsum
    assert L.pdae_colsum_det_workspace_bytes(8, 64) == 0
    n = L.pdae_colsum_det_workspace_bytes(32 * 64 * 64, 64)
    assert n > 0 and n % (64 * 4) == 0
    assert L.pdae_colsum_det_workspace_bytes(0, 64) < 0
    assert L.pdae_colsum_det(p, i64(32 * 64 * 64), 64, p, p, i64(n - 4), None) == -1 and "workspace" in _err(L)
    assert L.pdae_colsum_det(None, i64(8), 64, p, None, i64(0), None) == -1
    # GroupNorm backward
    n = L.pdae_gn_bwd_sums_det_workspace_bytes(2, 16, 16, 64)
    assert n > 0 and n % (2 * 64 * 2 * 4) == 0
    assert L.pdae_gn_bwd_sums_det_workspace_bytes(2, 0, 16, 64) < 0
    assert L.pdae_gn_bwd_sums_det(p, 64, None, 0, p, p, 1, 0, 2, 16, 16, p, p, i64(n - 4), None) == -1 and "workspace" in _err(L)
    assert L.pdae_gn_bwd_sums_det(p, 48, None, 0, p, p, 1, 0, 2, 16, 16, p, p, i64(n), None) == -1 and "channels" in _err(L)
    assert L.pdae_gn_bwd_sums_det(p, 64, None, 0, p, p, 1, 3, 2, 16, 16, p, p, i64(n), None) == -1 and "resample" in _err(L)
    assert L.pdae_gn_bwd_coef_det_workspace_bytes(2, 64) == 2 * 2 * 64 * 4
    assert L.pdae_gn_bwd_coef_det_workspace_bytes(0, 64) < 0
    f = ctypes.c_float(1e-5)
    assert L.pdae_gn_bwd_coef_det(p, p, p, p, None, 0, None, 0, 2, 64, 256, f, p, p, p, None, 0, None, 0, p, i64(8), None) == -1
    assert "workspace" in _err(L)
    assert L.pdae_gn_bwd_coef_det(p, p, p, p, None, 0, None, 0, 2, 48, 256, f, p, p, p, None, 0, None, 0, p, i64(1 << 20),
                                  None) == -1
    assert L.pdae_embedding_bwd_det(p, p, p, 4, 64, 0, None) == -1
    # tensor-core weight gradient plans
    assert L.pdae_wgrad_tc_det_workspace_bytes(None) < 0
    assert L.pdae_wgrad_tc_set_deterministic(None, p, i64(0)) == -1


def test_backward_ops_are_switched_or_guarded():
    """Every tensor-core backward op is switched to its DET kernel by a deterministic plan; the CUDA-core reductions with
    atomics stay refused there (their *_det forms are recorded instead)."""
    assert {"wgrad_tc", "wgrad_tc_bf16", "wgrad_tc_bf16_s2", "gemm_tc2_major", "gemm_tc2_softmax_grad",
            "conv_tc2_s2_dgrad"} <= DET_OPS
    assert not DET_OPS & NONDET_OPS
    assert {"conv2d_wgrad_simt", "conv2d_dgrad_simt", "colsum", "gn_bwd_sums", "gn_bwd_coef", "embedding_bwd"} <= NONDET_OPS
    for fn in DET_OPS:
        assert set(det_entry_points(fn)) <= set(_native.EXPORTS), fn
    for fn in ("conv2d_wgrad_simt_det", "conv2d_dgrad_simt_det", "colsum_det", "gn_bwd_sums_det", "gn_bwd_coef_det",
               "embedding_bwd_det"):
        assert fn not in NONDET_OPS and "pdae_" + fn in _native.EXPORTS


@pytest.mark.parametrize("entry,cls,args", [("shiftunet_train_forward", "ShiftUNetTrainer", 3),
                                            ("unet_train_forward", "UNetTrainer", 3),
                                            ("encoder_train_forward", "EncoderTrainer", 1)])
def test_trainer_caches_are_keyed_by_the_switch(entry, cls, args, monkeypatch):
    """Turning the switch on and off reuses both trainers; the deterministic one is built with det=True."""
    from pdae_b200 import train
    made = []

    class FakeTrainer:
        def __init__(self, net, B, H, W, amp=False, det=False):
            made.append(det)
            self.det = det
            self.params = []
            self.fwd = self.bwd = self

        def stale(self):
            return False

    monkeypatch.setattr(train, cls, FakeTrainer)
    for fn in ("_ShiftUNetFn", "_UNetFn", "_EncoderFn"):
        monkeypatch.setattr(getattr(train, fn), "apply", staticmethod(lambda tr, *a: tr))

    class Net(torch.nn.Module):
        def _shift_parts(self):
            return []

    net, x = Net(), torch.zeros(2, 3, 8, 8)
    call = lambda: getattr(train, entry)(net, x, *([None] * (args - 1)))
    was = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(False)
        a = call()
        torch.use_deterministic_algorithms(True, warn_only=True)
        b = call()
        torch.use_deterministic_algorithms(False)
        assert call() is a
        torch.use_deterministic_algorithms(True)
        assert call() is b
    finally:
        torch.use_deterministic_algorithms(was)
    assert made == [False, True] and not a.det and b.det
