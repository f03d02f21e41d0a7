"""torch.use_deterministic_algorithms on the GPU: under the switch every forward, sampling loop and metric gives the same bits
for the same inputs -- repeated forwards of one plan and of a fresh copy of the module, the graphed loops against the generic
loops, repeated calls of the gap measure, trajectory interpolation and metrics -- in every precision, while staying within
the golden tolerances; with the switch off the modules record the default plans again; a training step warns once."""
import copy
import warnings

import pytest
import torch

from tests import cases
from tests.configs import FFHQ_LATENT
from tests.test_gpu_parity import check
from tests.util import load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
PRECISIONS = ["fp32", "bf16", "bf16x3"]
SHIFT64 = load_golden("model_shiftunet_b64")[0]["cfg"]
UNET64 = {k: v for k, v in SHIFT64.items() if k != "latent_dim"}
FFHQ = {k: v for k, v in FFHQ_LATENT.items() if k != "model"}


@pytest.fixture(autouse=True)
def deterministic():
    was, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn_only)


def _equal(a, b, what):
    if isinstance(a, (tuple, list)):
        for k, (x, y) in enumerate(zip(a, b)):
            _equal(x, y, f"{what}[{k}]")
        return
    if not isinstance(a, torch.Tensor):
        assert a == b, f"{what}: {a!r} != {b!r}"
        return
    assert torch.equal(a, b), f"{what}: max |d| = {float((a.float() - b.float()).abs().max()):.3e}"


def _gd(cfg=None):
    from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
    return GaussianDiffusion(cfg or cases.DIFF, DEV)


def _module(kind, precision, cfg=None):
    from pdae_b200.model.mlp_skip_net import MLPSkipNet
    from pdae_b200.model.representation_learning.encoder import CELEBA64Encoder, FFHQEncoder
    from pdae_b200.model.shift_unet import ShiftUNet
    from pdae_b200.model.unet import UNet
    from pdae_b200.utils.synth import fill_module_
    m = {"shift": lambda: ShiftUNet(**SHIFT64), "unet": lambda: UNet(**UNET64), "enc64": lambda: CELEBA64Encoder(latent_dim=512),
         "enc128": lambda: FFHQEncoder(latent_dim=512), "mlp": lambda: MLPSkipNet(**(cfg or FFHQ))}[kind]()
    m = fill_module_(m, seed=31).eval().to(DEV)
    m.precision = precision
    return m


def _inputs(kind, B, size=None):
    from pdae_b200.utils.synth import synth_images, synth_normal
    if kind in ("enc64", "enc128"):
        return (synth_images(B, 3, 64 if kind == "enc64" else 128, 40).to(DEV),)
    t = torch.arange(B, dtype=torch.int64, device=DEV) * 37 % 1000
    if kind == "mlp":
        return synth_normal((B, 512), 41).to(DEV), t
    x = synth_normal((B, 3, size, size), 42).to(DEV)
    if kind == "shift":
        return x, t, synth_normal((B, 512), 43).to(DEV)
    return x, t


FORWARDS = [("shift", 4, 64),    # 64 x 64: one image spans 32 conv_tc3 tiles and several CTAs
            ("shift", 2, 16),    # the 8 x 8 level: two images per conv_tc2 tile
            ("unet", 4, 64),
            ("enc64", 4, None), ("enc128", 4, None),   # stride-2 convs and the split-K Linear
            ("mlp", 8, None), ("mlp", 256, None)]      # latent split-K at both batch sizes


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("kind,B,size", FORWARDS)
def test_repeated_forwards_are_bitwise_equal(kind, B, size, precision):
    m = _module(kind, precision)
    inp = _inputs(kind, B, size)
    with torch.no_grad():
        a = m(*inp)
        b = m(*inp)
        c = copy.deepcopy(m)(*inp)       # a fresh module records its own plan
    _equal(b, a, f"{kind} B={B} {precision}: second forward")
    _equal(c, a, f"{kind} B={B} {precision}: fresh copy")
    for plan, _ in m._plans().values():
        assert plan.det


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", ["model_shiftunet_b64", "model_unet_class", "model_encoder_celeba64", "model_encoder_ffhq128",
                                  "model_mlp_skip"])
def test_golden_tolerances_hold(name, precision):
    cfg, g = load_golden(name)
    m, inp = cases.model_case(cfg)
    m = m.cuda()
    m.precision = precision
    i = {k: v.cuda() for k, v in inp.items()}
    with torch.no_grad():
        if cfg["kind"] == "unet":
            check(m(i["x"], g["t"].cuda(), g["cond"].cuda() if "cond" in g else None), g["y"], precision, name)
        elif cfg["kind"] == "shiftunet":
            eps, grad = m(i["x"], g["t"].cuda(), i["z"])
            check(eps, g["eps"], precision, name + ".eps")
            check(grad, g["grad"], precision, name + ".grad")
        elif cfg["kind"] == "encoder":
            check(m(i["x"]), g["z"], precision, name)
        else:
            check(m(i["x"], g["t"].cuda()), g["y"], precision, name)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_graphed_ddim_loops_equal_generic(precision):
    m = _module("shift", precision)
    x, _, z = _inputs("shift", 2, 16)
    dd = _gd()._ddim("ddim10")
    with torch.no_grad():
        for loop in ("shift_ddim_sample_loop", "shift_ddim_encode_loop"):
            fast = getattr(dd, loop)(m, z, x)
            slow = getattr(dd, loop)(lambda a, b, c: m(a, b, c), z, x)
            _equal(fast, slow, f"{loop} {precision}: graphed vs generic")


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("kind", ["unet", "shift"])
def test_graphed_ddpm_loops_equal_generic(kind, precision):
    m = _module(kind, precision)
    x, _, *rest = _inputs(kind, 2, 16)
    d = _gd({"timesteps": 20, "betas_type": "linear"})
    out = []
    for generic in (False, True):
        cases.CpuStream(11, DEV).install(d)       # the same draws for both loops
        net = (lambda a, b, c: m(a, b, c)) if generic else m
        with torch.no_grad():
            out.append(d.representation_learning_ddpm_sample(None, net, x, x, rest[0]) if kind == "shift"
                       else d.regular_ddpm_sample(net, x, None))
    _equal(out[0], out[1], f"{kind} {precision}: graphed vs generic DDPM")


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("B", [8, 256])
def test_graphed_latent_loop_equals_generic(B, precision):
    from pdae_b200.diffusion.ddim import DDIM
    m = _module("mlp", precision)
    d = _gd()
    nb, tmap = d.get_ddim_betas_and_timestep_map("ddim100", d.latent_diffusion_config["alphas_cumprod"].cpu().numpy())
    dd = DDIM(nb, tmap, DEV)
    zT = _inputs("mlp", B)[0]
    with torch.no_grad():
        graphed = dd.latent_ddim_sample_loop(m, zT)
        generic = dd.latent_ddim_sample_loop(lambda a, b, c=None: m(a, b), zT)
    _equal(graphed, generic, f"latent ddim100 B={B} {precision}: graphed vs generic")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_repeat_calls_of_gap_interpolation_and_metrics(precision):
    from pdae_b200.metric import utils as metric
    from pdae_b200.utils.synth import synth_images
    m = _module("shift", precision)
    x0 = synth_images(2, 3, 16, 50).to(DEV)
    _, _, z = _inputs("shift", 2, 16)
    gaps = []
    for _ in range(2):
        d = _gd({"timesteps": 20, "betas_type": "linear"})
        cases.CpuStream(9, DEV).install(d)
        with torch.no_grad():
            gaps.append(d.representation_learning_gap_measure(lambda x: z, m, x0))
    _equal(gaps[0], gaps[1], f"gap measure {precision}")
    dd = _gd()._ddim("ddim10")
    with torch.no_grad():
        i1 = dd.shift_ddim_trajectory_interpolation(m, z, z.flip(1), x0, 0.3)
        i2 = dd.shift_ddim_trajectory_interpolation(m, z, z.flip(1), x0, 0.3)
    _equal(i1, i2, f"trajectory interpolation {precision}")
    a, b = synth_images(16, 3, 64, 51).to(DEV), synth_images(16, 3, 64, 52).to(DEV)
    _equal(metric.calculate_mse(a, b), metric.calculate_mse(a, b), "calculate_mse")
    _equal(metric.calculate_ssim(a, b), metric.calculate_ssim(a, b), "calculate_ssim")
    # the deterministic kernels' values against the default kernels (switch off) and, for the MSE, float64; the second shape
    # (40 x 40) has partial SSIM tiles and a per-image element count that is not a multiple of the MSE block
    c, e = synth_images(5, 3, 40, 53).to(DEV), synth_images(5, 3, 40, 54).to(DEV)
    for x, y in ((a, b), (c, e)):
        torch.use_deterministic_algorithms(True, warn_only=True)
        det_mse, det_ssim = metric.calculate_mse(x, y), metric.calculate_ssim(x, y)
        torch.use_deterministic_algorithms(False)
        torch.testing.assert_close(det_mse, metric.calculate_mse(x, y), rtol=1e-6, atol=0)
        torch.testing.assert_close(det_ssim, metric.calculate_ssim(x, y), rtol=1e-6, atol=1e-7)
        ref = (x.double() - y.double()).square().flatten(1).mean(1).float()
        torch.testing.assert_close(det_mse, ref, rtol=1e-5, atol=0)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_switch_off_returns_to_the_default_plans(precision):
    fresh = _module("shift", precision)
    toggled = copy.deepcopy(fresh)
    inp = _inputs("shift", 2, 16)
    with torch.no_grad():
        toggled(*inp)                                  # a deterministic plan
        torch.use_deterministic_algorithms(False)
        toggled(*inp)
        fresh(*inp)
    det = [p for p, _ in toggled._plans().values() if p.det]
    plain = [p for p, _ in toggled._plans().values() if not p.det]
    ref = [p for p, _ in fresh._plans().values()]
    assert len(det) == len(plain) == len(ref) == 1
    assert [fn for fn, _ in plain[0].ops] == [fn for fn, _ in ref[0].ops]
    assert [fn for fn, _ in det[0].ops] != [fn for fn, _ in ref[0].ops]


def test_training_step_warns_once_and_runs():
    m = _module("mlp", "fp32", cfg=load_golden("model_mlp_skip")[0]["cfg"]).train()
    x, t = _inputs("mlp", 4)[0][:, :64].contiguous(), _inputs("mlp", 4)[1]
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        for _ in range(2):
            y = m(x, t)
            y.square().mean().backward()
    msgs = [str(r.message) for r in w if "no deterministic implementation" in str(r.message)]
    assert len(msgs) == 1, msgs
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters() if p.requires_grad)
