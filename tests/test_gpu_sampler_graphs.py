"""The DDPM ancestral loops and DDIM trajectory interpolation on the one-graph-per-step path: the graph is really replayed,
each fused / standalone update is bitwise the arithmetic of the generic loop, whole loops match the generic loop (the network
wrapped in a lambda) and the CPU oracle, the random draws are unchanged, and nothing stays switched on afterwards."""
import collections
import ctypes

import pytest
import torch

from tests import cases
from tests.util import assert_close, load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
DDPM20 = {"timesteps": 20, "betas_type": "linear"}
TOL = {"fp32": dict(rtol=1e-3, atol=2e-4), "bf16x3": dict(rtol=1e-3, atol=2e-3)}   # graphed vs generic loop
LOOP = dict(rtol=1e-3, atol=2e-3)                                                   # vs the CPU oracle (test_gpu_glue)
SHIFT64 = load_golden("model_shiftunet_b64")[0]["cfg"]          # base 64: the image heads take the tensor-core path
UNET64 = {k: v for k, v in SHIFT64.items() if k != "latent_dim"}
UNETS = {"unet": UNET64, "sigma": dict(UNET64, learn_sigma=True), "class": dict(UNET64, num_class=10)}


def _gd(cfg=DDPM20):
    from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
    return GaussianDiffusion(cfg, DEV)


def _net(kind, cfg, precision):
    m, _ = cases.model_case({"kind": "shiftunet" if kind == "shift" else "unet", "cfg": cfg, "size": 16})
    sd = cases.sd_of(m)
    m = m.cuda().eval()
    m.precision = precision
    return m, sd


class Draws(cases.CpuStream):
    """CpuStream that records the shape of every randn call."""

    def __init__(self, seed):
        super().__init__(seed, DEV)
        self.calls = []

    def randn(self, shape):
        self.calls.append(tuple(shape))
        return super().randn(shape)


def _ddpm(d, m, kind, xT, cond, generic):
    net = (lambda a, b, c: m(a, b, c)) if generic else m
    with torch.no_grad():
        if kind == "shift":
            return d.representation_learning_ddpm_sample(None, net, xT, xT, cond)
        return d.regular_ddpm_sample(net, xT, cond)


def _inputs(kind, B=2, size=16):
    from pdae_b200.utils.synth import synth_normal
    xT = synth_normal((B, 3, size, size), 25).to(DEV)
    cond = {"shift": synth_normal((B, 512), 27).to(DEV), "class": torch.tensor([3, 7][:B], device=DEV)}.get(kind)
    return xT, cond


def _plan_io(m, kind, B, H, W):
    """(plan, x_in, t_in, eps, grad) of the plan a DDPM loop over `m` replays."""
    if kind == "shift":
        plan, (x_in, t_in, _, eps, grad) = m.plan_for(B, H, W)
        return plan, x_in, t_in, eps, grad
    plan, (x_in, t_in, _, eps) = m.plan_for(B, H, W)
    return plan, x_in, t_in, eps, None


# ---- 1. the fast path is taken --------------------------------------------------------------------------------------------
def test_graph_replayed_not_the_launch_loop(monkeypatch):
    from pdae_b200.engine import Plan
    calls = collections.Counter()
    orig = Plan._launch_all

    def spy(self, idx=None):
        calls["main" if idx is None else "prologue"] += 1
        return orig(self, idx)
    monkeypatch.setattr(Plan, "_launch_all", spy)
    d = _gd()
    for kind in ("unet", "shift"):
        m, _ = _net(kind, SHIFT64 if kind == "shift" else UNET64, "bf16x3")
        xT, cond = _inputs(kind)
        cases.CpuStream(1, DEV).install(d)
        m(xT, torch.zeros(2, dtype=torch.int64, device=DEV), *([cond] if cond is not None else []))   # record the plan first
        calls.clear()
        _ddpm(d, m, kind, xT, cond, generic=False)
        assert calls["main"] == 2, (kind, calls)            # warm-up + capture, not one per step
        _ddpm(d, m, kind, xT, cond, generic=False)
        assert calls["main"] == 2, (kind, calls)            # the captured graph is reused
        plan = _plan_io(m, kind, 2, 16, 16)[0]
        ent = [e for k, e in plan._step_cache.items() if k[1] == "ddpm"]
        assert len(ent) == 1 and ent[0].get("graph_fused") is not None, kind
    m, _ = _net("shift", SHIFT64, "bf16x3")
    xT, z = _inputs("shift")
    calls.clear()
    with torch.no_grad():
        _gd().representation_learning_ddim_trajectory_interpolation("ddim10", m, z, z.flip(0), xT, 0.3)
    assert calls["main"] == 2, calls
    plan, _ = m.plan_for_interp(2, 16, 16)
    assert any(k[1] == "interp" and e.get("graph_fused") is not None for k, e in plan._step_cache.items())


# ---- 2. each update is exact ----------------------------------------------------------------------------------------------
def _fused_vs_standalone(run, x, i, noise=None):
    """One graphed step with the update fused into the head epilogue, then the standalone update on the same x_t and on that
    step's own output buffers: must be bitwise equal."""
    run.begin()
    try:
        assert run.fused
        run.x_in.tensor.copy_(x)
        if noise is not None:
            run.noise.copy_(noise)
        run.seek(i)
        run.step()
        fused = run.x_in.tensor.clone()
        run.x_in.tensor.copy_(x)
        run._update()
        torch.cuda.synchronize()
        assert torch.equal(fused, run.x_in.tensor), f"step {i}: max diff {(fused - run.x_in.tensor).abs().max().item():.3e}"
    finally:
        run.end()


@pytest.mark.parametrize("kind", ["unet", "shift"])
def test_ddpm_fused_epilogue_bitwise(kind):
    from pdae_b200.diffusion.ddim import _DDPMRunner
    from pdae_b200.utils.synth import synth_normal
    d = _gd()
    m, _ = _net(kind, SHIFT64 if kind == "shift" else UNET64, "bf16x3")
    xT, z = _inputs(kind)
    plan, x_in, t_in, eps, grad = _plan_io(m, kind, 2, 16, 16)
    if kind == "shift":
        m.plan_for(2, 16, 16)[1][2].tensor.copy_(z)
    with torch.no_grad():
        for i in (13, 0):        # t == 0: no noise term
            run = _DDPMRunner(d, plan, x_in, t_in, eps, grad, 3)
            _fused_vs_standalone(run, xT, i, synth_normal(tuple(xT.shape), 40 + i).to(DEV))


@pytest.mark.parametrize("alpha", [0.0, 0.3, 1.0])
def test_interpolation_fused_epilogue_bitwise(alpha):
    from pdae_b200.diffusion.ddim import _InterpRunner
    dd = _gd(cases.DIFF)._ddim("ddim10")
    m, _ = _net("shift", SHIFT64, "bf16x3")
    xT, z = _inputs("shift")
    plan, (x_in, t_in, z1, z2, eps, g1, g2) = m.plan_for_interp(2, 16, 16)
    z1.tensor.copy_(z)
    z2.tensor.copy_(z.flip(0))
    with torch.no_grad():
        for i in (10, 4):
            _fused_vs_standalone(_InterpRunner(dd, plan, x_in, t_in, eps, g1, g2, 3, alpha), xT, i)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def test_standalone_kernels_match_generic_torch_expressions_bitwise():
    """pdae_noise_p_sample_shift (shift term; learned sigma read from a 2C output) and pdae_grad_blend against the torch
    expressions + pdae_noise_p_sample of the generic loops."""
    from pdae_b200 import _native
    from pdae_b200.utils.synth import synth_normal
    L, d = _native.lib(), _gd(cases.DIFF)
    d._log_betas = torch.log(d.betas)
    B, C, H, W = 4, 3, 8, 8
    per = C * H * W
    x, grad, noise = (synth_normal((B, C, H, W), s).to(DEV) for s in (71, 72, 73))
    out2 = synth_normal((B, 2 * C, H, W), 74).to(DEV)
    out2[:, C:].clamp_(-1, 1)
    t = torch.tensor([0, 1, 500, 999], device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run(eps, grad_, lr, eps_ld):
        y = torch.empty_like(x)
        rc = L.pdae_noise_p_sample_shift(_ptr(x), _ptr(eps), _ptr(grad_) if grad_ is not None else None, _ptr(d.shift_coef),
                                         _ptr(noise), lr, eps_ld, _ptr(t), _ptr(d.noise_posterior_mean_x_t_coef),
                                         _ptr(d.noise_posterior_mean_noise_coef), _ptr(d.posterior_log_variance_clipped),
                                         _ptr(d._log_betas), _ptr(y), B, per, st)
        _native.check(rc, "pdae_noise_p_sample_shift")
        return y
    eps = out2[:, :C].contiguous()
    want = d.noise_p_sample(x, t, eps + d.extract_coef_at_t(d.shift_coef, t, x.shape) * grad, noise=noise)
    assert torch.equal(run(eps, grad, None, per), want), "shift term"
    e, lr = torch.split(out2, C, dim=1)
    want = d.noise_p_sample(x, t, e, lr, noise=noise)
    got = run(out2, None, ctypes.c_void_p(out2.data_ptr() + per * 4), 2 * per)
    assert torch.equal(got, want), "learned sigma"
    assert torch.equal(run(eps, None, None, per), d.noise_p_sample(x, t, eps, noise=noise)), "plain"
    for alpha in (0.0, 0.3, 1.0, 0.7):
        ab = torch.tensor([1.0 - alpha, alpha], dtype=torch.float32, device=DEV)
        y = torch.empty_like(x)
        _native.check(L.pdae_grad_blend(_ptr(grad), _ptr(noise), _ptr(ab), _ptr(y), y.numel(), st), "pdae_grad_blend")
        assert torch.equal(y, (1.0 - alpha) * grad + alpha * noise), alpha


# ---- 3 + 4. whole loops, draws ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["unet", "sigma", "class", "shift"])
def test_ddpm_loops_match_generic_and_oracle(kind):
    from oracle import pdae_oracle as O
    D = O.DiffusionOracle(DDPM20)
    xT, cond = _inputs(kind)
    ref = None
    for precision in ("fp32", "bf16x3"):
        cfg = SHIFT64 if kind == "shift" else UNETS[kind]
        m, sd = _net(kind, cfg, precision)
        d = _gd()
        fast_draws = Draws(11)
        fast_draws.install(d)
        fast = _ddpm(d, m, kind, xT, cond, generic=False)
        slow_draws = Draws(11)          # (re-seeds the CPU generator)
        slow_draws.install(d)
        slow = _ddpm(d, m, kind, xT, cond, generic=True)
        assert fast_draws.calls == slow_draws.calls == [tuple(xT.shape)] * DDPM20["timesteps"]
        assert_close(fast, slow, what=f"{kind} {precision}: graphed vs generic DDPM", **TOL[precision])
        if ref is None:
            if kind == "shift":
                ref = D.ddpm_sample(lambda x, t, z: O.shiftunet_forward(sd, cfg, x, t, z), xT.cpu(), cases.CpuStream(11).randn,
                                    z=cond.cpu())
            else:
                ref = D.ddpm_sample(lambda x, t, c: O.unet_forward(sd, cfg, x, t, c), xT.cpu(), cases.CpuStream(11).randn,
                                    condition=cond.cpu() if cond is not None else None)
        assert_close(fast, ref, what=f"{kind} {precision}: graphed DDPM vs oracle", **LOOP)
        _check_switched_off(m, precision)


@pytest.mark.parametrize("B,size", [(2, 16), (1, 64)])
def test_interpolation_loop_matches_generic_and_oracle(B, size):
    from oracle import pdae_oracle as O
    D = O.DiffusionOracle(cases.DIFF)
    xT, z = _inputs("shift", B, size)
    z2 = z.flip(1)
    ref = None
    for precision in ("fp32", "bf16x3"):
        m, sd = _net("shift", SHIFT64, precision)
        dd = _gd(cases.DIFF)._ddim("ddim10")
        with torch.no_grad():
            fast = dd.shift_ddim_trajectory_interpolation(m, z, z2, xT, 0.3)
            slow = dd.shift_ddim_trajectory_interpolation(lambda a, b, c: m(a, b, c), z, z2, xT, 0.3)
        assert_close(fast, slow, what=f"B={B} {size}px {precision}: graphed vs generic interpolation", **TOL[precision])
        if ref is None:
            ref = D.trajectory_interpolation("ddim10", lambda x, t, zz: O.shiftunet_forward(sd, SHIFT64, x, t, zz), z.cpu(),
                                             z2.cpu(), xT.cpu(), 0.3)
        assert_close(fast, ref, what=f"B={B} {size}px {precision}: graphed interpolation vs oracle", **LOOP)
        if size == 16:
            _check_switched_off(m, precision)


# ---- 5. the frozen half runs once in interpolation ------------------------------------------------------------------------
def test_interpolation_plan_records_frozen_half_once():
    m, _ = _net("shift", SHIFT64, "bf16x3")
    count = lambda plan: collections.Counter(fn for fn, _ in plan.ops)
    one, eps_only, interp = (count(m.plan_for(2, 16, 16)[0]), count(m.plan_for(2, 16, 16, with_shift=False)[0]),
                             count(m.plan_for_interp(2, 16, 16)[0]))
    # one pass = frozen half F + shift half S (+ its z prologue); epsilon-only = F; interpolation = F + 2 S
    want = collections.Counter({k: 2 * one[k] - eps_only[k] for k in one})
    assert interp == +want, (interp, want)
    assert sum(interp.values()) < 2 * sum(one.values())
    assert list(m.plan_for_interp(2, 16, 16)[0].head_fuse) == ["grad"]


# ---- 6. nothing stays switched on ------------------------------------------------------------------------------------------
def _check_switched_off(m, precision):
    for plan, _ in m._plans().values():
        for buf in plan.head_fuse.values():
            assert not buf.tensor.any(), "fusion descriptor must be switched off after the loop"
    if hasattr(m, "latent_dim") and precision == "bf16x3":
        from tests.test_gpu_parity import check
        cfg, g = load_golden("model_shiftunet_b64")
        _, inp = cases.model_case(cfg)
        with torch.no_grad():
            e1, g1 = m(inp["x"].cuda(), g["t"].cuda(), inp["z"].cuda())
        check(e1, g["eps"], "bf16x3", "forward after the graphed loops (eps)")
        check(g1, g["grad"], "bf16x3", "forward after the graphed loops (grad)")


# ---- 7. the native plan executor -------------------------------------------------------------------------------------------
def test_native_plan_executor(monkeypatch):
    monkeypatch.setenv("PDAE_NATIVE_PLAN", "1")
    m, _ = _net("unet", UNET64, "bf16x3")
    xT, _ = _inputs("unet")
    d = _gd()
    cases.CpuStream(5, DEV).install(d)
    fast = _ddpm(d, m, "unet", xT, None, generic=False)
    assert m.plan_for(2, 16, 16)[0]._native_plans, "plan not on the native executor"
    cases.CpuStream(5, DEV).install(d)
    slow = _ddpm(d, m, "unet", xT, None, generic=True)
    assert_close(fast, slow, what="native plan: graphed vs generic DDPM", **TOL["bf16x3"])
    m, _ = _net("shift", SHIFT64, "bf16x3")
    xT, z = _inputs("shift")
    dd = _gd(cases.DIFF)._ddim("ddim10")
    with torch.no_grad():
        fast = dd.shift_ddim_trajectory_interpolation(m, z, z.flip(0), xT, 0.3)
        slow = dd.shift_ddim_trajectory_interpolation(lambda a, b, c: m(a, b, c), z, z.flip(0), xT, 0.3)
    assert m.plan_for_interp(2, 16, 16)[0]._native_plans
    assert_close(fast, slow, what="native plan: graphed vs generic interpolation", **TOL["bf16x3"])
