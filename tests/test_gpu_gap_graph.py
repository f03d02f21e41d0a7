"""The gap measure (GaussianDiffusion.representation_learning_gap_measure) on the one-graph-per-step path: the graph is really
replayed, pdae_gap_terms matches float64 means of the generic loop's fp32 element expressions and is bitwise repeatable, the
graphed lists match the generic loop (the decoder wrapped in a lambda) with unchanged random draws, nothing stays switched on,
other decoders and grad mode keep the generic loop, and graphs are reused or recorded correctly across calls."""
import collections
import ctypes

import numpy as np
import pytest
import torch

from tests import cases
from tests.test_gpu_sampler_graphs import SHIFT64, _check_switched_off, _net
from tests.util import assert_close

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
GAP20 = {"timesteps": 20, "betas_type": "linear"}
TOL = {"fp32": dict(rtol=1e-4, atol=1e-9), "bf16x3": dict(rtol=1e-3, atol=1e-9)}   # graphed vs generic gap lists


def _gd(cfg=GAP20):
    from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
    return GaussianDiffusion(cfg, DEV)


class RandDraws(cases.CpuStream):
    """CpuStream that records the shape of every rand_like call."""

    def __init__(self, seed):
        super().__init__(seed, DEV)
        self.calls = []

    def rand_like(self, x):
        self.calls.append(tuple(x.shape))
        return super().rand_like(x)


def _inputs(B, size=16, seed=0):
    from pdae_b200.utils.synth import synth_images, synth_normal
    return synth_images(B, 3, size, 60 + seed).to(DEV), synth_normal((B, 512), 70 + seed).to(DEV)


def _gap(d, m, x0, z, seed=9, generic=False):
    """(gap_pred, gap_ae, rand_like shapes) of one gap measure on `d` with a fresh seeded draw stream."""
    draws = RandDraws(seed)
    draws.install(d)
    net = (lambda a, b, c: m(a, b, c)) if generic else m
    with torch.no_grad():
        gp, ga = d.representation_learning_gap_measure(lambda x: z, net, x0)
    return gp, ga, draws.calls


def _spy_graphed(monkeypatch):
    from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
    calls = collections.Counter()
    orig = GaussianDiffusion._gap_graphed

    def spy(self, *a, **k):
        calls["graphed"] += 1
        return orig(self, *a, **k)
    monkeypatch.setattr(GaussianDiffusion, "_gap_graphed", spy)
    return calls


# ---- 1. the fast path is taken --------------------------------------------------------------------------------------------
def test_graph_replayed_not_the_launch_loop(monkeypatch):
    from pdae_b200.engine import Plan
    calls = collections.Counter()
    orig = Plan._launch_all

    def spy(self, idx=None):
        calls["main" if idx is None else "prologue"] += 1
        return orig(self, idx)
    monkeypatch.setattr(Plan, "_launch_all", spy)
    m, _ = _net("shift", SHIFT64, "bf16x3")
    x0, z = _inputs(2)
    with torch.no_grad():
        m(x0, torch.zeros(2, dtype=torch.int64, device=DEV), z)     # record the plan first
    d = _gd()
    calls.clear()
    gp, ga, _ = _gap(d, m, x0, z)
    assert calls["main"] == 2, calls                     # warm-up + capture, not one per step
    assert len(gp) == len(ga) == GAP20["timesteps"]
    _gap(d, m, x0, z)
    assert calls["main"] == 2, calls                     # the captured graph is reused
    plan = m.plan_for(2, 16, 16)[0]
    ent = [e for k, e in plan._step_cache.items() if k[1] == "gap"]
    assert len(ent) == 1 and ent[0].get("graph") is not None and ent[0].get("graph_fused") is None


# ---- 2. the kernel ---------------------------------------------------------------------------------------------------------
def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize("B,per", [(1, 7), (1, 3 * 4096 + 5), (3, 3 * 37 * 41), (2, 3 * 128 * 128)])
def test_gap_terms_kernel_vs_float64(B, per):
    """pdae_gap_terms against float64 means of the generic loop's fp32 torch expressions (per-sample t indexes the tables,
    t[0] picks the row); two runs are bitwise equal and no other row is written."""
    from pdae_b200 import _native
    from pdae_b200.utils.synth import synth_normal
    L, d = _native.lib(), _gd(cases.DIFF)
    x0, xt, eps, grad = (synth_normal((B, per), s).to(DEV) for s in (81, 82, 83, 84))
    ws = torch.empty(L.pdae_gap_terms_workspace_bytes(B * per) // 8, dtype=torch.float64, device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for ts in ([0] * B, [517] * B, [999] * B, [3, 400, 999][:B]):
        t = torch.tensor(ts, dtype=torch.int64, device=DEV)

        def run():
            out = torch.full((1000, 2), float("nan"), device=DEV)
            rc = L.pdae_gap_terms(_ptr(x0), _ptr(xt), _ptr(eps), _ptr(grad), _ptr(t), _ptr(d.x_0_posterior_mean_x_0_coef),
                                  _ptr(d.x_0_posterior_mean_x_t_coef), _ptr(d.sqrt_recip_alphas_cumprod),
                                  _ptr(d.sqrt_recip_alphas_cumprod_m1), _ptr(d.shift_coef), _ptr(ws), ws.numel() * 8, _ptr(out),
                                  B, per, st)
            _native.check(rc, "pdae_gap_terms")
            return out
        out, again = run(), run()
        row = ts[0]
        assert torch.equal(out[row], again[row]), f"t={ts}: not bitwise repeatable"
        s = x0.shape
        true = d.q_posterior_mean(x0, xt, t)
        m1 = d.q_posterior_mean(d.predicted_noise_to_predicted_x_0(xt, t, eps), xt, t)
        eps_ae = eps + d.extract_coef_at_t(d.shift_coef, t, s) * grad
        m2 = d.q_posterior_mean(d.predicted_noise_to_predicted_x_0(xt, t, eps_ae), xt, t)
        want = torch.stack([((true - m1) ** 2).double().mean(), ((true - m2) ** 2).double().mean()])
        rel = ((out[row].double() - want).abs() / want.abs()).max().item()
        assert rel <= 1e-6, f"B={B} per={per} t={ts}: rel {rel:.3e} ({out[row].tolist()} vs {want.tolist()})"
        others = torch.cat([out[:row], out[row + 1:]])
        assert torch.isnan(others).all(), "rows other than t[0] written"


# ---- 3 + 4. graphed against generic, draws -------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [2, 3])
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_graphed_matches_generic_and_draws(precision, B):
    m, _ = _net("shift", SHIFT64, precision)
    x0, z = _inputs(B)
    d = _gd()
    fp, fa, fast_calls = _gap(d, m, x0, z, seed=13)
    sp, sa, slow_calls = _gap(d, m, x0, z, seed=13, generic=True)
    assert fast_calls == slow_calls == [tuple(x0.shape)] * GAP20["timesteps"]
    assert all(isinstance(v, float) for v in fp + fa)
    np.testing.assert_allclose(fp, sp, **TOL[precision], err_msg=f"{precision} B={B}: gap_pred")
    np.testing.assert_allclose(fa, sa, **TOL[precision], err_msg=f"{precision} B={B}: gap_ae")
    _check_switched_off(m, precision)


# ---- 5. nothing stays switched on ------------------------------------------------------------------------------------------
def test_plain_forward_unchanged_after_gap_measure():
    m, _ = _net("shift", SHIFT64, "bf16x3")
    x0, z = _inputs(2)
    t = torch.tensor([3, 11], dtype=torch.int64, device=DEV)
    with torch.no_grad():
        e0, g0 = m(x0, t, z)
    _gap(_gd(), m, x0, z)
    with torch.no_grad():
        e1, g1 = m(x0, t, z)
    # two bf16x3 forwards of one plan are not bitwise equal (fp32 atomics in the statistics), hence a tolerance
    assert_close(e1, e0, rtol=1e-3, atol=1e-4, what="eps after the gap measure")
    assert_close(g1, g0, rtol=1e-3, atol=1e-4, what="grad after the gap measure")
    for plan, _ in m._plans().values():
        for buf in plan.head_fuse.values():
            assert not buf.tensor.any(), "fusion descriptor must stay off"


# ---- 6. fallbacks ---------------------------------------------------------------------------------------------------------
def test_fallbacks_take_the_generic_loop(monkeypatch):
    calls = _spy_graphed(monkeypatch)
    m, _ = _net("shift", SHIFT64, "bf16x3")
    x0, z = _inputs(2)
    d = _gd()
    ref_p, ref_a, _ = _gap(d, m, x0, z)
    assert calls["graphed"] == 1
    gp, ga, _ = _gap(d, m, x0, z, generic=True)           # a lambda-wrapped decoder
    assert calls["graphed"] == 1
    np.testing.assert_allclose(gp, ref_p, **TOL["bf16x3"])
    for p in m.parameters():
        p.requires_grad_(False)                            # grad mode on, but the decoder's inference forward
    RandDraws(9).install(d)
    with torch.enable_grad():
        gp, ga = d.representation_learning_gap_measure(lambda x: z, m, x0)
    assert calls["graphed"] == 1
    np.testing.assert_allclose(gp, ref_p, **TOL["bf16x3"])
    np.testing.assert_allclose(ga, ref_a, **TOL["bf16x3"])
    sigma, _ = _net("shift", dict(SHIFT64, learn_sigma=True), "bf16x3")
    assert sigma.output_channel == 6
    with pytest.raises(RuntimeError):                      # the reference's expression does not broadcast for 2C outputs
        _gap(d, sigma, x0, z)
    assert calls["graphed"] == 1


# ---- 7. reuse across calls -------------------------------------------------------------------------------------------------
def test_second_call_other_input_and_batch(monkeypatch):
    calls = _spy_graphed(monkeypatch)
    m, _ = _net("shift", SHIFT64, "bf16x3")
    d = _gd()
    for B, seed in ((2, 0), (3, 1), (2, 2)):
        x0, z = _inputs(B, seed=seed)
        fp, fa, _ = _gap(d, m, x0, z, seed=20 + seed)
        sp, sa, _ = _gap(d, m, x0, z, seed=20 + seed, generic=True)
        np.testing.assert_allclose(fp, sp, **TOL["bf16x3"], err_msg=f"B={B} seed={seed}: gap_pred")
        np.testing.assert_allclose(fa, sa, **TOL["bf16x3"], err_msg=f"B={B} seed={seed}: gap_ae")
    assert calls["graphed"] == 3
    graphs = {B: [e["graph"] for k, e in m.plan_for(B, 16, 16)[0]._step_cache.items() if k[1] == "gap"] for B in (2, 3)}
    assert len(graphs[2]) == len(graphs[3]) == 1 and graphs[2][0] is not graphs[3][0]
