"""Deterministic plans without a GPU: the deterministic kernels contain no float atomic in their SASS, their entry points
refuse bad arguments before any launch, and a plan recorded under torch.use_deterministic_algorithms holds none of the atomic
ops."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from pdae_b200 import _native
from pdae_b200.engine import DET_OPS, NONDET_OPS, Buf, Plan, _STREAM

# what nvcc 12.9 emits for sm_90a: fp32 / fp32x2 / fp64 global reductions and atomics, and the CAS loop of a shared-memory
# float atomicAdd
FLOAT_ATOMICS = ("REDG.E.ADD.F32", "REDG.E.ADD.F32x2", "REDG.E.ADD.F64", "ATOMG.E.ADD.F32", "ATOMG.E.ADD.F64",
                 "ATOMS.CAST.SPIN")
DET_KERNELS = {
    # (mangled-name pattern, instances expected)
    r"conv_tc2_kernel.*Lb1EE": 10,        # DET = true: BN 64/128/256 x out dtype, stride-2 forward x 4, split-K x 2 ... (>=)
    r"conv_tc3_kernel.*Lb1EE": 8,         # DET = true: BN x split mode x out dtype
    r"stem_conv_bf16_kernelILi\dELi\dELb1E": 8,
    r"mse_kernelILb1E": 1,
    r"ssim_kernelILb1E": 1,
    r"ch_parts_kernel": 1,
    r"stat_parts_reduce_kernel": 1,
    r"gn_group_reduce_kernel": 1,
    r"finish_parts_kernel": 1,
    r"splitk_reduce_kernel": 1,
}


def _functions():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _native.LIB_PATH], capture_output=True, text=True).stdout
    out = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        out[name.strip()] = body
    return out


def _atomics(body):
    """The float-atomic mnemonics in a function's SASS.  A mnemonic is a prefix of the instruction's full name (nvcc 12.9
    writes e.g. REDG.E.ADD.F32.FTZ.RN.STRONG.GPU), so it must end at a '.', whitespace or the end of the token."""
    return {m for m in FLOAT_ATOMICS if re.search(re.escape(m) + r"(?=[.\s;]|$)", body, re.M)}


def test_deterministic_kernels_have_no_float_atomics():
    funcs = _functions()
    for pat, n in DET_KERNELS.items():
        hits = [f for f in funcs if re.search(pat, f)]
        assert len(hits) >= n, (pat, hits)
        for f in hits:
            assert not _atomics(funcs[f]), (f, _atomics(funcs[f]))
    # the same matcher sees each family in the default kernels that the deterministic ones replace
    def found(pat):
        return set().union(*[_atomics(b) for f, b in funcs.items() if re.search(pat, f)])
    assert "REDG.E.ADD.F32" in found(r"conv_tc3_kernelILi128ELb0ELb1ELb0EE")       # conv_tc3<128, bf16, bf16 out, default>
    assert "REDG.E.ADD.F32x2" in found(r"conv_tc2_kernelILi128ELb0ELi0ELi16ELb0EE")  # the default split-K Linear
    assert "REDG.E.ADD.F64" in found(r"mse_kernelILb0E")
    assert "ATOMS.CAST.SPIN" in found(r"ch_stats_kernel")
    assert "REDG.E.ADD.F64" in found(r"gn_stats_kernel")


def _err(L):
    return L.pdae_last_error().decode()


def test_entry_points_reject_bad_arguments_before_any_launch():
    """Dummy pointers are never dereferenced: every call below fails its argument checks."""
    L = _native.lib()
    p = ctypes.c_void_p(16)
    assert L.pdae_stats_det_workspace_bytes(0, 64, 64) < 0
    assert L.pdae_stats_det_workspace_bytes(2, 64, 64) > 0
    assert L.pdae_ch_stats_det(None, 2, 64, 64, p, p, 1 << 20, None) == -1
    assert L.pdae_ch_stats_det(p, 2, 64, 64, p, p, 8, None) == -1 and "workspace" in _err(L)
    assert L.pdae_ch_stats_det(p, 2, 64, 66, p, p, 1 << 20, None) == -1
    assert L.pdae_gn_stats_det(p, 48, None, 0, 2, 64, p, p, 1 << 20, None) == -1 and "% 32" in _err(L)
    assert L.pdae_gn_stats_det(p, 64, None, 0, 2, 64, p, p, 8, None) == -1 and "workspace" in _err(L)
    assert L.pdae_conv_tc2_set_deterministic(None, p, 0) == -1
    assert L.pdae_conv_tc3_set_deterministic(None, p, 0) == -1
    assert L.pdae_conv_tc2_det_workspace_bytes(None) < 0 and L.pdae_conv_tc3_det_workspace_bytes(None) < 0
    assert L.pdae_stem_conv_det_workspace_bytes(2, 64, 64, 64, 3) < 0
    need = L.pdae_stem_conv_det_workspace_bytes(2, 64, 64, 64, 1)
    assert need > 0
    assert L.pdae_stem_conv_bf16_det(p, p, None, p, p, 2, 64, 64, 3, 64, 3, p, need, None) == -1 and "stride" in _err(L)
    assert L.pdae_stem_conv_bf16_det(p, p, None, p, p, 2, 64, 64, 3, 64, 1, p, need - 8, None) == -1 and "workspace" in _err(L)
    assert L.pdae_stem_conv_bf16_det(p, p, None, p, p, 2, 64, 64, 4, 256, 1, p, 1 << 30, None) == -1 and "shared" in _err(L)
    assert L.pdae_stem_conv_bf16_det(p, p, None, p, None, 2, 64, 64, 3, 64, 1, p, need, None) == -1
    assert L.pdae_mse_det_workspace_bytes(0, 10) < 0
    n = L.pdae_mse_det_workspace_bytes(4, 3 * 64 * 64)
    assert n == 4 * 6 * 8
    assert L.pdae_mse_per_image_det(p, p, 4, 3 * 64 * 64, p, n - 8, p, None) == -1 and "workspace" in _err(L)
    assert L.pdae_mse_per_image_det(p, None, 4, 3 * 64 * 64, p, n, p, None) == -1
    n = L.pdae_ssim_det_workspace_bytes(4, 3, 64, 64)
    assert n == 4 * 3 * 4 * 4 * 8
    assert L.pdae_ssim_per_image_det(p, p, p, 4, 3, 64, 64, p, n - 8, p, None) == -1 and "workspace" in _err(L)
    assert L.pdae_ssim_per_image_det(p, p, None, 4, 3, 64, 64, p, n, p, None) == -1


class CpuPlan(Plan):
    """A plan recorded from CPU parameters: the recording and buffer logic of Plan without its CUDA checks (such a plan is
    never finalised or run)."""

    def param(self, p):
        if p is None:
            return None
        self.params.append((p, p.data_ptr()))
        return Buf(p.shape, p.dtype, p.detach())

    def pack(self, key, sources, fn):
        if key not in self._pack_cache:
            self._pack_cache[key] = Buf(*(lambda t: (t.shape, t.dtype, t))(fn().contiguous()))
        return self._pack_cache[key]


def _modules():
    from pdae_b200.model.mlp_skip_net import MLPSkipNet
    from pdae_b200.model.representation_learning.encoder import CELEBA64Encoder, FFHQEncoder
    from pdae_b200.model.shift_unet import ShiftUNet
    from pdae_b200.model.unet import UNet
    from pdae_b200.utils.synth import fill_module_
    from tests.configs import FFHQ_LATENT
    from tests.util import load_golden
    shift = load_golden("model_shiftunet_b64")[0]["cfg"]
    unet = {k: v for k, v in shift.items() if k != "latent_dim"}
    s, u = fill_module_(ShiftUNet(**shift), seed=1).eval(), fill_module_(UNet(**unet), seed=2).eval()
    e64, e128 = fill_module_(CELEBA64Encoder(latent_dim=512), seed=3).eval(), fill_module_(FFHQEncoder(latent_dim=512), seed=4).eval()
    mlp = fill_module_(MLPSkipNet(**{k: v for k, v in FFHQ_LATENT.items() if k != "model"}), seed=5).eval()
    return [("shiftunet 64px", s, lambda P: s._build(P, 4, 64, 64, True)),
            ("shiftunet 16px", s, lambda P: s._build(P, 2, 16, 16, True)),
            ("shiftunet interp", s, lambda P: s._build(P, 2, 16, 16, interp=True)),
            ("unet 64px", u, lambda P: u._build(P, 4, 64, 64)),
            ("encoder 64px", e64, lambda P: e64._build(P, 4, 64, 64)),
            ("encoder 128px", e128, lambda P: e128._build(P, 4, 128, 128)),
            ("mlp", mlp, lambda P: mlp._build(P, 8)),
            ("mlp one_t", mlp, lambda P: mlp._build(P, 256, one_t=True))]


@pytest.mark.parametrize("precision", ["fp32", "bf16", "bf16x3"])
def test_module_plans_recorded_under_the_switch_hold_no_atomic_ops(precision, monkeypatch):
    """Every module's real plan builder, recorded as a deterministic plan: none of the atomic ops, and every tensor-core op is
    one that finalize switches to its DET kernels."""
    from pdae_b200.model.module import PlannedModule
    monkeypatch.setattr(PlannedModule, "_device", lambda self: torch.device("cpu"))
    for name, m, build in _modules():
        m.precision = precision
        P = CpuPlan(torch.device("cpu"), precision, check_device=False, deterministic=True)
        build(P)
        ops = [fn for fn, _ in P.ops]
        assert not NONDET_OPS & set(ops), (name, sorted(NONDET_OPS & set(ops)))
        tc = {fn for fn in ops if fn.startswith(("conv_tc", "gemm_tc"))}
        assert tc <= DET_OPS, (name, sorted(tc - DET_OPS))
        if precision != "fp32" and not name.startswith("mlp"):
            assert tc, name    # the tensor-core modes do run tensor-core ops here
        assert P._stats_elems == 0, name   # no zeroed statistics arena
        if precision == "fp32" and "net" in name:
            assert "gn_stats_det" in ops, name
        if precision == "bf16" and name.startswith("encoder"):
            assert {"stem_conv_bf16_det", "conv_tc2_s2", "conv_tc2_splitk"} <= set(ops), name
        if precision != "fp32" and name == "shiftunet 64px":
            assert "conv_tc3" in ops, name


def test_finalize_refuses_an_atomic_op_in_a_deterministic_plan():
    P = Plan(torch.device("cpu"), "bf16", check_device=False, deterministic=True)
    x = P.new((2, 16, 16, 64), name="x")
    x.keep = True
    P.call("ch_stats", x, 2, 256, 64, P.new((2, 64, 2)), _STREAM)
    with pytest.raises(ValueError, match="float atomics"):
        P.finalize()


def test_module_plan_cache_is_keyed_by_the_switch():
    """_get_plan keys its cache by the switch: turning it on and off reuses both plans."""
    from pdae_b200.model.module import PlannedModule

    class M(PlannedModule):
        def _device(self):
            return torch.device("cpu")

    import pdae_b200.model.module as mod
    made = []

    class FakePlan:
        def __init__(self, dev, prec, deterministic=False):
            made.append(deterministic)
            self.det = deterministic

        def finalize(self):
            return self

        def stale(self):
            return False

    real = mod.Plan
    mod.Plan = FakePlan
    was = torch.are_deterministic_algorithms_enabled()
    try:
        m = M()
        a = m._get_plan(("k",), lambda P: None)[0]
        torch.use_deterministic_algorithms(True)
        b = m._get_plan(("k",), lambda P: None)[0]
        torch.use_deterministic_algorithms(False)
        assert m._get_plan(("k",), lambda P: None)[0] is a
        torch.use_deterministic_algorithms(True, warn_only=True)
        assert m._get_plan(("k",), lambda P: None)[0] is b
    finally:
        torch.use_deterministic_algorithms(was)
        mod.Plan = real
    assert made == [False, True] and not a.det and b.det
