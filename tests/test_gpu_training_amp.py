"""Training under torch.autocast (the reference trainers' `enable_amp`, trainer/train_representation_learning.py:48-49,94,
111-116): the single-pass bf16 wgrad_tc kernel through the C-ABI, the bf16 ShiftUNet / UNet training plans against oracle
autograd on the CPU, the plans actually recorded, fp16 autocast and GradScaler, and full-precision steps interleaved with AMP
steps on one module."""
import copy
import ctypes

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import pdae_oracle as O
from pdae_b200 import _native
from tests import cases
from tests.test_gpu_wgrad_tc import CASES as WGRAD_CASES
from tests.util import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"

# every trainable conv of this ShiftUNet except the 3-channel head is tensor-core eligible (channels 64 / 128, 32x32 images)
SHIFT_CFG = dict(input_channel=3, base_channel=64, channel_multiplier=[1, 2, 2], num_residual_blocks_of_a_block=1,
                 attention_resolutions=[2], num_heads=1, head_channel=-1, use_new_attention_order=False, dropout=0.0,
                 latent_dim=512)
UNET_CFG = {k: v for k, v in SHIFT_CFG.items() if k != "latent_dim"}
SIZE, B = 32, 2
T_STEPS = torch.tensor([7, 805])
SPLIT_OPS = ("gn_apply_split3", "qkv_split3", "softmax_split3", "wgrad_tc")


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


# ---- 1. the kernel ---------------------------------------------------------------------------------------------------
def run_wgrad_bf16(B, H, W, Cin, Cout, k, seed=0):
    g = torch.Generator(device="cpu").manual_seed(77 + seed)
    act = (torch.randn(B, H, W, Cin, generator=g) * 1.3 + 0.2).to(DEV).to(torch.bfloat16).contiguous()
    dy = (torch.randn(B, H, W, Cout, generator=g) * 0.05).to(DEV).to(torch.bfloat16).contiguous()
    dw = torch.zeros(k * k, Cin, Cout, device=DEV)
    L = _native.lib()
    assert L.pdae_wgrad_tc_supported(H, W, Cin, Cout, k)
    h = ctypes.c_void_p()
    _native.check(L.pdae_wgrad_tc_create_bf16(ctypes.byref(h), _p(act), _p(dy), _p(dw), B, H, W, Cin, Cout, k),
                  "pdae_wgrad_tc_create_bf16")
    try:
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _native.check(L.pdae_wgrad_tc_run(h, st), "pdae_wgrad_tc_run")
        torch.cuda.synchronize()
    finally:
        L.pdae_wgrad_tc_destroy(h)
    # float64 autograd of the bf16-ROUNDED operands: the kernel's products are exact, only the fp32 summation order differs
    x = act.double().permute(0, 3, 1, 2)
    w = torch.zeros(Cout, Cin, k, k, device=DEV, dtype=torch.float64, requires_grad=True)
    F.conv2d(x, w, padding=k // 2).backward(dy.double().permute(0, 3, 1, 2))
    ref = w.grad.reshape(Cout, Cin, k * k).permute(2, 1, 0)            # [tap][cin][cout]
    return dw.double(), ref


@pytest.mark.parametrize("B,H,W,Cin,Cout,k", WGRAD_CASES)
def test_wgrad_tc_bf16_matches_float64_autograd_of_rounded_operands(B, H, W, Cin, Cout, k):
    got, ref = run_wgrad_bf16(B, H, W, Cin, Cout, k)
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    assert err <= 2e-5 * scale + 1e-7, (err, scale)


# ---- helpers -----------------------------------------------------------------------------------------------------------
def _gd():
    from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
    return GaussianDiffusion(cases.DIFF, torch.device(DEV))


def _shift_module(seed=6):
    from pdae_b200.model.shift_unet import ShiftUNet
    from pdae_b200.utils.synth import fill_module_
    return fill_module_(ShiftUNet(**SHIFT_CFG), seed=seed)


def _to_train(dec):
    dec = dec.cuda().train()
    dec.freeze()
    dec.set_train_mode()
    dec.precision = "fp32"
    return dec


def _shift_inputs():
    from pdae_b200.utils.synth import synth_images, synth_normal
    x0 = synth_images(B, 3, SIZE, 31)
    noise = torch.randn(x0.shape, generator=torch.Generator().manual_seed(3))
    z = synth_normal((B, SHIFT_CFG["latent_dim"]), 17)
    return x0, noise, z


def _shift_loss(gd, dec, x0, t, noise, z):
    """representation_learning_train_one_batch (gaussian_diffusion.py:234-255) with the latent z given as a leaf."""
    x_t = gd.q_sample(x0, t, noise)
    eps, grad = dec(x_t, t, z)
    s = x0.shape
    target = eps + gd.extract_coef_at_t(gd.shift_coef, t, s) * grad
    return gd.p_loss(noise, target, weight=gd.extract_coef_at_t(gd.weight, t, s))


def _shift_step(gd, dec, inputs, autocast_dtype=None, enabled=True):
    """One forward + backward; returns (loss, {name: grad}, z grad) and clears the gradients."""
    x0, noise, z = inputs
    zl = z.cuda().requires_grad_(True)
    if autocast_dtype is None:
        loss = _shift_loss(gd, dec, x0.cuda(), T_STEPS.cuda(), noise.cuda(), zl)
    else:
        with torch.autocast("cuda", dtype=autocast_dtype, enabled=enabled):
            loss = _shift_loss(gd, dec, x0.cuda(), T_STEPS.cuda(), noise.cuda(), zl)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in dec.named_parameters() if p.grad is not None}
    for p in dec.parameters():
        p.grad = None
    return loss.detach(), grads, zl.grad.detach().clone()


def _check_grads(named_grads, ref_grads, what, rel=5e-2, floor=2e-3):
    """Per tensor: rel-L2 <= rel, or max|err| <= rel * max|ref| + floor * (largest gradient entry of the step): biases and
    weights of a GroupNorm have small gradients made of large cancelling sums."""
    assert sorted(named_grads) == sorted(ref_grads)
    gmax = max(float(g.abs().max()) for g in ref_grads.values())
    bad, worst, worst_big, worst_abs = [], (0.0, ""), (0.0, ""), 0.0
    for k, ref in ref_grads.items():
        got, ref = named_grads[k].double().cpu(), ref.double().cpu()
        r = rel_l2(got, ref)
        err = float((got - ref).abs().max())
        ref_max = float(ref.abs().max())
        worst, worst_abs = max(worst, (r, k)), max(worst_abs, err / gmax)
        if ref_max > 0.1 * gmax:         # the tensors that carry the bulk of the gradient
            worst_big = max(worst_big, (r, k))
        if r > rel and err > rel * ref_max + floor * gmax:
            bad.append((k, tuple(ref.shape), round(r, 4), f"err={err:.2e} ref_max={ref_max:.2e}"))
    print(f"{what}: largest |grad| {gmax:.3e}; worst rel-L2 {worst[0]:.2e} ({worst[1]}); among tensors with max|grad| > 10% "
          f"of the largest {worst_big[0]:.2e} ({worst_big[1]}); worst max|err| / largest |grad| {worst_abs:.2e}")
    assert not bad, f"{what}: gradients off: " + "; ".join(map(str, bad[:30]))


def _amp_trainer(net):
    trs = [tr for tr in net._train_cache.values() if tr.amp]
    assert len(trs) == 1, len(trs)
    return trs[0]


def _assert_bf16_plans(plans):
    from pdae_b200.engine import PDAE_BF16
    n_wgrad = 0
    for P in plans:
        for fn, args in P.ops:
            assert fn not in SPLIT_OPS, fn
            if fn == "conv_tc2":
                assert not args[0].split3, "split-operand conv_tc2 in an AMP plan"
            if fn == "conv_tc3":
                assert args[4] == PDAE_BF16, "split-operand conv_tc3 in an AMP plan"
            n_wgrad += fn == "wgrad_tc_bf16"
    return n_wgrad


# ---- 2. + 3. PDAE step under bf16 autocast ---------------------------------------------------------------------------
def test_pdae_step_under_bf16_autocast_matches_oracle_and_runs_bf16_plans():
    dec0 = _shift_module()
    inputs = _shift_inputs()
    x0, noise, z = inputs
    dsd = {k: v.requires_grad_(k.startswith(("label_emb", "shift_"))) for k, v in cases.sd_of(dec0).items()}
    zr = z.clone().requires_grad_(True)
    ref_loss = O.DiffusionOracle(cases.DIFF).representation_learning_loss(
        lambda x: zr, lambda x, t, zz: O.shiftunet_forward(dsd, SHIFT_CFG, x, t, zz), x0, T_STEPS, noise)
    ref_loss.backward()
    dec = _to_train(dec0)
    loss, grads, gz = _shift_step(_gd(), dec, inputs, torch.bfloat16)
    ref_loss = ref_loss.detach()
    r = abs(float(loss) - float(ref_loss)) / abs(float(ref_loss))
    print(f"bf16 autocast PDAE step: loss {float(loss):.6f} vs oracle {float(ref_loss):.6f} (rel {r:.2e})")
    assert r <= 1e-2
    ref = {k: v.grad for k, v in dsd.items() if v.grad is not None}
    _check_grads(dict(grads, z=gz), dict(ref, z=zr.grad), "ShiftUNet bf16 autocast vs oracle")
    # 3. the bf16 plans really ran: no split-operand op anywhere, one bf16 wgrad per eligible trainable conv
    tr = _amp_trainer(dec)
    assert tr.frozen.precision == "bf16" and tr.bwd.precision == "bf16" and tr.fwd.train_tc == "bf16"
    L = _native.lib()
    eligible = 0
    for part in dec._shift_parts():
        for m in part.modules():
            if isinstance(m, (nn.Conv1d, nn.Conv2d)):
                co, ci, k = m.weight.shape[0], m.weight.shape[1], m.weight.shape[2]
                eligible += co % 64 == 0 and ci % 64 == 0 and k in (1, 3)
    lab = dec.label_emb
    eligible += bool(L.pdae_wgrad_tc_supported(1, 1, lab.in_features, lab.out_features, 1))
    assert eligible >= 10
    assert _assert_bf16_plans([tr.frozen, tr.fwd, tr.bwd]) == eligible


# ---- 4. + 5. fp16 autocast and GradScaler ------------------------------------------------------------------------------
# Two runs of the same step are not bitwise equal, with or without autocast: the GroupNorm backward, the split-K weight
# gradients and the forward's GroupNorm statistics are sums of fp32 atomics.  In the bf16 step the next bf16 rounding turns a
# rare last-bit difference into a one-ulp bf16 difference, so two bf16 runs differ by up to ~1.4e-2 rel-L2 on a small
# GroupNorm gradient (H100 measurement); the fp32-grade step differs by ~2e-5.  Same-step comparisons use these spreads.
AMP_SPREAD = dict(rel=5e-2, floor=2e-3)
FP32_SPREAD = dict(rel=1e-4, floor=2e-5)


def test_fp16_autocast_and_grad_scaler_use_the_bf16_plans():
    gd = _gd()
    dec = _to_train(_shift_module())
    inputs = _shift_inputs()
    loss_b, g_b, gz_b = _shift_step(gd, dec, inputs, torch.bfloat16)
    tr = _amp_trainer(dec)
    loss_h, g_h, gz_h = _shift_step(gd, dec, inputs, torch.float16)
    assert _amp_trainer(dec) is tr and len(dec._train_cache) == 1      # either autocast dtype: the same bf16 trainer
    print(f"fp16 vs bf16 autocast: loss {float(loss_h):.7f} vs {float(loss_b):.7f}")
    assert abs(float(loss_h) - float(loss_b)) <= 1e-3 * abs(float(loss_b))
    _check_grads(dict(g_h, z=gz_h), dict(g_b, z=gz_b), "fp16 vs bf16 autocast", **AMP_SPREAD)
    # the reference trainer's sequence: scaler.scale(loss).backward(); scaler.step(opt); scaler.update()
    scaler = torch.amp.GradScaler("cuda")
    params = [p for p in dec.parameters() if p.requires_grad]
    opt = torch.optim.Adam(params, lr=1e-4)
    x0, noise, z = inputs
    zl = z.cuda().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.float16):
        loss = _shift_loss(gd, dec, x0.cuda(), T_STEPS.cuda(), noise.cuda(), zl)
    scaler.scale(loss).backward()
    scale = float(scaler.get_scale())
    assert _amp_trainer(dec) is tr and scale > 1
    named = dict(dec.named_parameters())
    assert all(torch.isfinite(named[k].grad).all() for k in g_b)
    unscaled = {k: named[k].grad / scale for k in g_b}
    # a power-of-two scale is exact in bf16 and fp32: scaled / scale differs from the unscaled step only by the run spread
    _check_grads(dict(unscaled, z=zl.grad / scale), dict(g_b, z=gz_b), f"GradScaler (scale {scale:g}) grads / scale vs unscaled",
                 **AMP_SPREAD)
    norm = sum(float(g.double().norm()) ** 2 for g in unscaled.values()) ** 0.5
    norm_b = sum(float(g.double().norm()) ** 2 for g in g_b.values()) ** 0.5
    assert abs(norm / norm_b - 1) <= 1e-2, (norm, norm_b)
    before = [p.detach().clone() for p in params]
    scaler.step(opt)
    scaler.update()
    assert any(not torch.equal(p, q) for p, q in zip(params, before)), "GradScaler skipped a finite step"


# ---- 6. full-precision steps interleaved with AMP steps ----------------------------------------------------------------
def test_alternating_amp_and_full_precision_steps():
    gd = _gd()
    dec = _to_train(_shift_module())
    fresh = copy.deepcopy(dec)            # never sees autocast
    inputs = _shift_inputs()
    _, g_ref, gz_ref = _shift_step(gd, fresh, inputs)
    _, g_amp1, gz_amp1 = _shift_step(gd, dec, inputs, torch.bfloat16)
    _, g_full, gz_full = _shift_step(gd, dec, inputs)
    _, g_amp2, gz_amp2 = _shift_step(gd, dec, inputs, torch.bfloat16)
    assert len(dec._train_cache) == 2      # one full-precision and one AMP trainer, each with its own buffers
    full_tr = [tr for tr in dec._train_cache.values() if not tr.amp][0]
    _, g_off, gz_off = _shift_step(gd, dec, inputs, torch.bfloat16, enabled=False)
    assert len(dec._train_cache) == 2 and [tr for tr in dec._train_cache.values() if not tr.amp][0] is full_tr
    fresh_tr = list(fresh._train_cache.values())[0]
    assert not fresh_tr.amp
    # the full-precision trainer of the module that saw autocast records exactly the plans of one that never did
    for a, b in ((full_tr.frozen, fresh_tr.frozen), (full_tr.fwd, fresh_tr.fwd), (full_tr.bwd, fresh_tr.bwd)):
        assert a.precision == b.precision and a.train_tc == b.train_tc
        assert [(fn, [(x.shape, x.dtype) if hasattr(x, "shape") else None for x in args]) for fn, args in a.ops] == \
               [(fn, [(x.shape, x.dtype) if hasattr(x, "shape") else None for x in args]) for fn, args in b.ops]
    _check_grads(dict(g_full, z=gz_full), dict(g_ref, z=gz_ref), "full precision after AMP vs never-autocast module",
                 **FP32_SPREAD)
    _check_grads(dict(g_off, z=gz_off), dict(g_ref, z=gz_ref), "autocast(enabled=False) vs never-autocast module",
                 **FP32_SPREAD)
    _check_grads(dict(g_amp2, z=gz_amp2), dict(g_amp1, z=gz_amp1), "AMP step after a full-precision step vs the first",
                 **AMP_SPREAD)


# ---- 7. regular DPM step (UNetTrainer) under bf16 autocast -------------------------------------------------------------
def test_regular_dpm_step_under_bf16_autocast_matches_oracle():
    from pdae_b200.model.unet import UNet
    from pdae_b200.utils.synth import fill_module_, synth_images
    net = fill_module_(UNet(**UNET_CFG), seed=5)
    x0 = synth_images(B, 3, SIZE, 32)
    noise = torch.randn(x0.shape, generator=torch.Generator().manual_seed(3))
    sd = {k: v.requires_grad_(True) for k, v in cases.sd_of(net).items()}
    D = O.DiffusionOracle(cases.DIFF)
    ref_loss = D.regular_loss(lambda x, tt, cc: O.unet_forward(sd, UNET_CFG, x, tt, cc), x0, T_STEPS, noise, None)
    ref_loss.backward()
    net = net.cuda().train()
    net.precision = "fp32"
    gd = _gd()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        x_t = gd.q_sample(x0.cuda(), T_STEPS.cuda(), noise.cuda())
        loss = gd.p_loss(noise.cuda(), net(x_t, T_STEPS.cuda(), None))
    got, want = float(loss.detach()), float(ref_loss.detach())
    r = abs(got - want) / abs(want)
    print(f"bf16 autocast regular step: loss {got:.6f} vs oracle {want:.6f} (rel {r:.2e})")
    assert r <= 1e-2
    loss.backward()
    grads = {k: p.grad for k, p in net.named_parameters() if p.grad is not None}
    ref = {k: v.grad for k, v in sd.items() if v.grad is not None}
    _check_grads(grads, ref, "UNet bf16 autocast vs oracle")
    tr = _amp_trainer(net)
    assert tr.bwd.precision == "bf16" and tr.fwd.train_tc == "bf16"
    assert _assert_bf16_plans([tr.fwd, tr.bwd]) > 0
