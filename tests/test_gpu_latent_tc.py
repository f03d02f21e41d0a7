"""The latent MLPSkipNet's sampling forward on the tensor cores ("bf16" / "bf16x3": split-operand Linears, fp32-grade) and the
latent DDIM loop as one CUDA graph per step: the split row kernels against the fp32 kernels bit for bit, the recorded plans,
the whole forward and the ddim100 loop against the CPU oracle, packed-weight refresh, the graphed loop against the standalone
update and the generic loop, the random draws of latent_diffusion_sample, and per-row forwards around a loop."""
import collections
import copy
import ctypes

import pytest
import torch

from oracle import pdae_oracle as O
from pdae_b200 import _native
from tests import cases
from tests.configs import FFHQ_LATENT
from tests.util import assert_close, load_golden, rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
FFHQ = {k: v for k, v in FFHQ_LATENT.items() if k != "model"}
ONE = dict(rtol=1e-3, atol=1e-4)            # one forward vs the oracle (the fp32 bound of test_gpu_configs)
TC = ("bf16", "bf16x3")


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rows(B, N, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(B, N, generator=g) * scale).to(DEV)


def _split(v):
    hi = v.to(torch.bfloat16)
    return hi, (v - hi.float()).to(torch.bfloat16)


def _mlp(cfg=FFHQ, seed=79, precision="bf16"):
    from pdae_b200.model.mlp_skip_net import MLPSkipNet
    from pdae_b200.utils.synth import fill_module_
    m = fill_module_(MLPSkipNet(**cfg), seed=seed).eval()
    sd = cases.sd_of(m)
    m = m.cuda()
    m.precision = precision
    return m, sd


def _ddim(style="ddim100"):
    from pdae_b200.diffusion.ddim import DDIM
    from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
    d = GaussianDiffusion(cases.DIFF, DEV)
    nb, tmap = d.get_ddim_betas_and_timestep_map(style, d.latent_diffusion_config["alphas_cumprod"].cpu().numpy())
    return DDIM(nb, tmap, DEV)


def _zT(B, D, seed=81):
    from pdae_b200.utils.synth import synth_normal
    return synth_normal((B, D), seed).clamp(-1, 1)


# ---- 1. split row kernels ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ln", [True, False])
@pytest.mark.parametrize("cond_ld", [-1, 0, 256, 1024])   # -1: no cond; 0: one shared cond row; 1024: block at column 256
def test_split_kernels_are_the_split_of_the_fp32_kernels(ln, cond_ld):
    B, N, D = 7, 256, 128
    ld, col0 = N + D + 64, 64                                 # the written columns sit inside wider blocks
    L = _native.lib()
    h = _rows(B, N, 1, 2.0)
    bank = _rows(B if cond_ld > 0 else 1, max(cond_ld, N), 2, 0.5) if cond_ld >= 0 else None
    off = 256 if cond_ld > N else 0
    if cond_ld < 0:
        cond_c, cptr, cld = None, None, 0
    else:
        cond_c = bank[:, off:off + N].expand(B, N).contiguous()       # what the fp32 kernel reads
        cptr, cld = ctypes.c_void_p(bank[:, off:].data_ptr()), cond_ld
    lw, lb = (_rows(1, N, 3).flatten() + 1, _rows(1, N, 4).flatten()) if ln else (None, None)
    ref = torch.empty(B, N, device=DEV)
    _native.check(L.pdae_mlp_mod_ln_act(_p(h), _p(cond_c), _p(lw), _p(lb), ctypes.c_float(1e-5), 1, _p(ref), N, B, N, _st()),
                  "mlp_mod_ln_act")
    sentinel = torch.tensor(-7.0, dtype=torch.bfloat16)
    got = torch.full((B, 3 * ld), float(sentinel), device=DEV, dtype=torch.bfloat16)
    _native.check(L.pdae_mlp_mod_ln_act_split3(_p(h), cptr, cld, _p(lw), _p(lb), ctypes.c_float(1e-5), 1, _p(got), ld, col0, B,
                                               N, _st()), "mlp_mod_ln_act_split3")
    z = _rows(B, D, 6)
    _native.check(L.pdae_copy_cols_split3(_p(z), _p(got), ld, col0 + N, B, D, _st()), "copy_cols_split3")
    torch.cuda.synchronize()
    blocks = got.view(B, 3, ld)
    for v, c0, n in ((ref, col0, N), (z, col0 + N, D)):
        hi, lo = _split(v)
        assert torch.equal(blocks[:, 0, c0:c0 + n], hi) and torch.equal(blocks[:, 2, c0:c0 + n], hi)
        assert torch.equal(blocks[:, 1, c0:c0 + n], lo)
    assert (blocks[:, :, :col0] == sentinel).all() and (blocks[:, :, col0 + N + D:] == sentinel).all()


# ---- 2. the plans -----------------------------------------------------------------------------------------------------------
def _ops(plan):
    return [fn for fn, _ in plan.ops]


def _parent_fp32_ops(n_layers):
    """The op list of the CUDA-core plan as it was recorded before the tensor-core plan existed."""
    ops = ["timestep_embedding", "conv2d_simt", "conv2d_simt", "copy_cols", "copy_cols"]
    ops += ["conv2d_simt", "conv2d_simt", "mlp_mod_ln_act"] * (n_layers - 1)
    return ops + ["conv2d_simt"]


@pytest.mark.parametrize("B", [3, 128])
def test_plans(B):
    n = FFHQ["num_layers"]
    m, _ = _mlp()
    m.precision = "fp32"
    plan, _ = m.plan_for(B)
    assert _ops(plan) == _parent_fp32_ops(n)
    assert m.plan_for(B, one_t=True)[0] is plan            # "fp32": the loop replays the per-row plan
    for prec in TC:
        m.precision = prec
        for one_t in (False, True):
            plan, _ = m.plan_for(B, one_t=one_t)
            ops = _ops(plan)
            assert ops.count("conv2d_simt") == 2, ops       # time_embed only
            assert ops.count("conv_tc2") + ops.count("conv_tc2_splitk") == n + 1, ops     # n Linears + ONE linear_emb bank
            assert ops.count("mlp_mod_ln_act_split3") == n, ops                          # bank operand + n - 1 layers
            assert ops.count("copy_cols_split3") == 3 and "mlp_mod_ln_act" not in ops and "copy_cols" not in ops
            te = [args for fn, args in plan.ops if fn == "timestep_embedding"][0]
            assert te[1] == (1 if one_t else B)             # the loop plan embeds one timestep
            row = [args for fn, args in plan.ops if fn == "mlp_mod_ln_act_split3"][1:]
            assert all(a[2] == (0 if one_t else 9 * FFHQ["model_channel"]) for a in row)    # cond_ld
        assert m.plan_for(B, one_t=True)[0] is not m.plan_for(B)[0]
    # a net whose widths are not multiples of 64 keeps the CUDA-core plan in every mode
    odd, _ = _mlp(dict(FFHQ, model_channel=200, num_layers=3), precision="bf16")
    assert _ops(odd.plan_for(4)[0]) == _parent_fp32_ops(3)


# ---- 3. whole forward vs the oracle -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", TC)
@pytest.mark.parametrize("B", [3, 8, 128, 200])
def test_forward_matches_oracle(precision, B):
    from pdae_b200.utils.synth import synth_normal
    m, sd = _mlp(precision=precision)
    z = synth_normal((B, FFHQ["input_channel"]), 80 + B)
    t = torch.linspace(0, 999, B).round().long()
    with torch.no_grad():
        ref = O.mlp_skip_net_forward(sd, FFHQ, z, t)
        y = m(z.cuda(), t.cuda())
    print(f"ffhq_latent forward {precision} B={B}: rel-L2 vs oracle {rel_l2(y, ref):.2e}")
    assert_close(y, ref, what=f"ffhq_latent {precision} B={B}", **ONE)
    assert "conv_tc2_splitk" in _ops(m.plan_for(B)[0])


# ---- 4. packed-weight refresh -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", TC)
def test_packed_weights_refresh(precision):
    from pdae_b200.utils.synth import synth_normal
    m, sd = _mlp(precision=precision)
    z, t = synth_normal((8, 512), 90), torch.tensor([0, 3, 40, 200, 500, 700, 950, 999])
    with torch.no_grad():
        m(z.cuda(), t.cuda())                                               # record + pack
        for p in (m.layers[3].linear.weight, m.layers[5].linear_emb.weight, m.layers[9].linear.bias):
            p.mul_(0.5)                                                     # in place: bumps the version
        y = m(z.cuda(), t.cuda())
    sd2 = cases.sd_of(m)
    assert_close(y, O.mlp_skip_net_forward(sd2, FFHQ, z, t), what="after an in-place update", **ONE)
    other, sd3 = _mlp(seed=5)
    with torch.no_grad():
        m.load_state_dict(other.state_dict())
        y = m(z.cuda(), t.cuda())
        assert_close(y, O.mlp_skip_net_forward(sd3, FFHQ, z, t), what="after load_state_dict", **ONE)
        m.layers[2].linear.weight.data.mul_(2.0)                            # .data: no version bump ...
        m.invalidate_packed()                                               # ... so the caller says so
        y = m(z.cuda(), t.cuda())
        assert_close(y, O.mlp_skip_net_forward(cases.sd_of(m), FFHQ, z, t), what="after invalidate_packed", **ONE)
        # a sampling loop re-packs at its start without being told
        m.layers[4].linear.weight.data.mul_(0.5)
        zT = _zT(4, 512)
        got = _ddim("ddim10").latent_ddim_sample_loop(m, zT.cuda())
    sd4 = cases.sd_of(m)
    ref = O.DiffusionOracle(cases.DIFF).latent_ddim_sample("ddim10", lambda zz, tt: O.mlp_skip_net_forward(sd4, FFHQ, zz, tt), zT)
    assert rel_l2(got, ref) <= 1e-4, rel_l2(got, ref)


# ---- 5. the graphed loop ----------------------------------------------------------------------------------------------------
def test_graph_replayed_not_the_launch_loop(monkeypatch):
    from pdae_b200.engine import Plan
    calls = collections.Counter()
    orig = Plan._launch_all

    def spy(self, idx=None):
        calls["main" if idx is None else "prologue"] += 1
        return orig(self, idx)
    monkeypatch.setattr(Plan, "_launch_all", spy)
    for prec in ("bf16", "bf16x3", "fp32"):
        m, _ = _mlp(precision=prec)
        d = _ddim("ddim10")
        zT = _zT(4, 512).cuda()
        calls.clear()
        with torch.no_grad():
            d.latent_ddim_sample_loop(m, zT)
            assert calls["main"] == 2, (prec, calls)       # warm-up + capture, not one per step
            d.latent_ddim_sample_loop(m, zT)
            assert calls["main"] == 2, (prec, calls)       # the captured graph is reused
        plan = m.plan_for(4, one_t=True)[0]
        assert [k[1] for k in plan._step_cache] == ["latent"] and list(plan._step_cache.values())[0]["graph"] is not None
    # autograd on, a CPU input, a 4-D input, another callable: the generic loop
    from pdae_b200.diffusion.ddim import graphable
    with torch.no_grad():
        assert graphable(m, zT) and not graphable(m, zT.cpu()) and not graphable(lambda a, b, c=None: m(a, b), zT)
        assert not graphable(m, zT[:, :, None, None])
    assert not graphable(m, zT)


@pytest.mark.parametrize("precision", ["bf16", "bf16x3", "fp32"])
def test_in_graph_update_is_the_standalone_ddim_step(precision):
    from pdae_b200.diffusion.ddim import _StepRunner
    m, _ = _mlp(precision=precision)
    d = _ddim("ddim100")
    B = 16
    plan, (x_in, t_in, eps) = m.plan_for(B, one_t=True)
    run = _StepRunner(d, plan, x_in, t_in, eps, None, "sample", 512, key=("latent",))
    z = _zT(B, 512, 7).cuda()
    with torch.no_grad():
        run.begin()
        try:
            for i in (100, 57, 1):
                x_in.tensor.copy_(z)
                run.seek(i)
                run.step()
                graphed = x_in.tensor.clone()
                t = torch.full((B,), i, device=DEV, dtype=torch.long)
                assert torch.equal(t_in.tensor, d.t_transform(t))
                ref = d._update(z, t, eps.tensor.clone(), None, "sample")
                assert torch.equal(graphed, ref), (precision, i)
        finally:
            run.end()


@pytest.mark.parametrize("precision", ["bf16", "bf16x3", "fp32"])
def test_graphed_loop_matches_generic_loop_and_oracle(precision):
    """Generic loop: the net wrapped in a lambda (per-step plan runs, per-row time embedding).  The two differ only by the
    order of the split-K partial sums (fp32 atomics) in the tensor-core modes; in "fp32" they are the same launches."""
    m, sd = _mlp(precision=precision)
    d = _ddim("ddim100")
    B = 16
    zT = _zT(B, 512)
    with torch.no_grad():
        graphed = d.latent_ddim_sample_loop(m, zT.cuda())
        generic = d.latent_ddim_sample_loop(lambda a, b, c=None: m(a, b), zT.cuda())
    ref = O.DiffusionOracle(cases.DIFF).latent_ddim_sample("ddim100", lambda zz, tt: O.mlp_skip_net_forward(sd, FFHQ, zz, tt), zT)
    e_gen, e_ref = rel_l2(graphed, generic), rel_l2(graphed, ref)
    print(f"latent ddim100 B={B} {precision}: graphed vs generic rel-L2 {e_gen:.2e}, "
          f"max|d| {float((graphed - generic).abs().max()):.2e}; vs CPU oracle rel-L2 {e_ref:.2e} (generic {rel_l2(generic, ref):.2e})")
    if precision == "fp32":
        assert torch.equal(graphed, generic)
    else:
        assert e_gen <= 1e-5, e_gen
    assert e_ref <= 1e-4, e_ref


@pytest.mark.parametrize("precision", TC)
def test_existing_latent_loop_fixture(precision):
    """The TINY_MLP ddim10 fixture at the fp32 bound, in the tensor-core modes, and at B = 64."""
    cfg, g = load_golden("loop_latent_ddim10")
    m, sd = _mlp(cfg["cfg"], seed=8, precision=precision)
    d = _ddim("ddim10")
    with torch.no_grad():
        out = d.latent_ddim_sample_loop(m, _zT(2, 64, 29).cuda())
    assert_close(out, g["z"], what="latent loop", **ONE)
    assert "conv_tc2_splitk" in _ops(m.plan_for(2, one_t=True)[0])
    zT = _zT(64, 64, 30)
    with torch.no_grad():
        out = d.latent_ddim_sample_loop(m, zT.cuda())
    ref = O.DiffusionOracle(cases.DIFF).latent_ddim_sample("ddim10", lambda zz, tt: O.mlp_skip_net_forward(sd, cfg["cfg"], zz, tt),
                                                           zT)
    excess = float(((out.cpu() - ref).abs() / (ONE["atol"] + ONE["rtol"] * ref.abs())).max())
    print(f"TINY_MLP ddim10 B=64 {precision}: rel-L2 vs oracle {rel_l2(out, ref):.2e}, worst element {excess:.2f} of the bound")
    assert rel_l2(out, ref) <= 1e-4, rel_l2(out, ref)


class _Wrapped:
    """Any latent callable that is not an MLPSkipNet (takes the generic loop)."""

    def __init__(self, m):
        self.m, self.input_channel = m, m.input_channel

    def __call__(self, z, t, cond=None):
        return self.m(z, t)


class _Draws(cases.CpuStream):
    def __init__(self, seed):
        super().__init__(seed, DEV)
        self.calls = []

    def randn(self, shape):
        self.calls.append(tuple(shape))
        return super().randn(shape)


@pytest.mark.parametrize("precision", TC)
def test_latent_diffusion_sample_draws_and_result(precision):
    from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
    i = {k: v.to(DEV) for k, v in cases.glue_inputs().items()}
    cfg, g = load_golden("glue_latent_sample")
    mlp, _ = cases.model_case({"kind": "mlp", "cfg": cfg["cfg_mlp"]})
    mlp = mlp.cuda().eval()
    mlp.precision = precision
    dec, _ = cases.model_case({"kind": "shiftunet", "cfg": cfg["cfg_shift"], "size": 16})
    dec = dec.cuda().eval()
    dec.precision = "fp32"
    outs, draws = [], []
    for fn in (mlp, _Wrapped(mlp)):
        s = _Draws(cfg["seed"])
        d = s.install(GaussianDiffusion(cases.DIFF, DEV))
        with torch.no_grad():
            outs.append(d.latent_diffusion_sample("ddim10", "ddim10", fn, dec, i["xT"], i["mean64"], i["std64"]))
        draws.append(s.calls)
    assert draws[0] == draws[1] and draws[0][0] == (2, 64), draws
    assert_close(outs[0], g["y"], rtol=1e-3, atol=2e-3, what="latent_diffusion_sample")
    assert_close(outs[0], outs[1], rtol=1e-3, atol=2e-3, what="graphed vs generic latent loop")


@pytest.mark.parametrize("precision", ["bf16", "bf16x3", "fp32"])
def test_per_row_forward_around_a_loop(precision):
    from pdae_b200.utils.synth import synth_normal
    """The loop records its own plan: the per-row plan, its buffers and its per-row time embedding are untouched.  In the
    tensor-core modes two calls of the same plan already differ by the order of the split-K partial sums (fp32 atomics),
    a few 1e-6 rel-L2 after ten layers; a forward reading another row's timestep or a clobbered buffer is off by far more."""
    m, sd = _mlp(precision=precision)
    B = 16
    z, t = synth_normal((B, 512), 95), torch.linspace(0, 999, B).round().long()
    with torch.no_grad():
        before = m(z.cuda(), t.cuda())
        again = m(z.cuda(), t.cuda())
        fwd_plan = m.plan_for(B)[0]
        _ddim("ddim10").latent_ddim_sample_loop(m, _zT(B, 512).cuda())
        after = m(z.cuda(), t.cuda())
    assert m.plan_for(B)[0] is fwd_plan
    print(f"per-row forward {precision}: repeat call rel-L2 {rel_l2(again, before):.2e}, after a loop {rel_l2(after, before):.2e}")
    if precision == "fp32":
        assert torch.equal(before, after)
    else:
        assert rel_l2(after, before) <= 2e-5, rel_l2(after, before)
        assert_close(after, O.mlp_skip_net_forward(sd, FFHQ, z, t), what="per-row forward after a loop", **ONE)


def test_native_plan_executor_runs_the_loop(monkeypatch):
    """The C-ABI plan executor (PDAE_NATIVE_PLAN=1) records and replays the new row kernels."""
    m, sd = _mlp(precision="bf16x3")
    ref_m = copy.deepcopy(m)
    zT = _zT(8, 512).cuda()
    d = _ddim("ddim10")
    with torch.no_grad():
        want = d.latent_ddim_sample_loop(ref_m, zT)
        monkeypatch.setenv("PDAE_NATIVE_PLAN", "1")
        got = d.latent_ddim_sample_loop(m, zT)
    assert m.plan_for(8, one_t=True)[0]._native_plans
    assert rel_l2(got, want) <= 1e-5, rel_l2(got, want)
