"""The semantic encoder under torch.autocast (the reference trainers' `enable_amp`, trainer/train_representation_learning.py:
48-49,94,111-116): the stride-2 bf16 tensor-core kernels through the C-ABI against float64 autograd, the encoder step and the
whole PDAE step against oracle autograd on the CPU, the plans actually recorded, fp16 autocast and GradScaler, and AMP steps
interleaved with full-precision steps on one encoder."""
import copy
import ctypes

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import pdae_oracle as O
from pdae_b200 import _native
from tests import cases
from tests.test_gpu_training_amp import AMP_SPREAD, FP32_SPREAD, T_STEPS, _check_grads, _gd, _shift_loss, _shift_module

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (input H = W, Cin, Cout) of every stride-2 conv of the 64-px and the 128-px encoders after the 3-channel stem
S2_SHAPES = [(32, 64, 128), (16, 128, 128), (8, 128, 128),
             (64, 64, 128), (32, 128, 256), (16, 256, 256), (8, 256, 256)]
S2_CASES = [(B,) + s for s in S2_SHAPES for B in (2, 32)]
SIMT_CONV_OPS = ("conv2d_simt", "conv2d_dgrad_simt", "conv2d_wgrad_simt")
ENC_KIND = {64: "celeba64", 128: "ffhq128"}


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _run(create, run, destroy, *args):
    L = _native.lib()
    h = ctypes.c_void_p()
    _native.check(getattr(L, create)(ctypes.byref(h), *args), create)
    try:
        _native.check(getattr(L, run)(h, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), run)
        torch.cuda.synchronize()
    finally:
        getattr(L, destroy)(h)


def _within(got, ref, what):
    scale = ref.abs().max().item()
    err = (got.double() - ref).abs().max().item()
    print(f"{what}: max|err| {err:.3e} = {err / scale:.2e} of max|ref| {scale:.3e}")
    assert torch.isfinite(got).all(), f"{what}: non-finite output (an element not written?)"
    assert err <= 2e-5 * scale, (what, err, scale)


# ---- 1. the kernels ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,Cin,Cout", S2_CASES)
def test_stride2_kernels_match_float64_autograd_of_rounded_operands(B, H, Cin, Cout):
    """Forward (+bias), data gradient and weight gradient of conv3x3(stride 2, pad 1) on bf16 operands, against float64
    F.conv2d and its autograd on the same bf16-rounded values: the products are exact, only the fp32 summation order differs."""
    W, Ho, Wo = H, H // 2, H // 2
    L = _native.lib()
    assert L.pdae_conv_s2_tc_supported(H, W, Cin, Cout)
    g = torch.Generator(device="cpu").manual_seed(H * 7 + Cin + B)
    x = (torch.randn(B, H, W, Cin, generator=g) * 1.3 + 0.2).to(DEV).to(torch.bfloat16).contiguous()
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (3 * Cin ** 0.5)).to(DEV).to(torch.bfloat16)
    bias = (torch.randn(Cout, generator=g) * 0.5).to(DEV)
    dy = (torch.randn(B, Ho, Wo, Cout, generator=g) * 0.05).to(DEV).to(torch.bfloat16).contiguous()
    x64 = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    w64 = w.double().requires_grad_(True)
    y64 = F.conv2d(x64, w64, bias.double(), stride=2, padding=1)
    y64.backward(dy.double().permute(0, 3, 1, 2))

    out = torch.full((B, Ho, Wo, Cout), float("nan"), device=DEV)
    wp = w.reshape(Cout, Cin, 9).permute(2, 0, 1).contiguous()                 # [tap][Cout][Cin]
    _run("pdae_conv_tc2_create_s2", "pdae_conv_tc2_run", "pdae_conv_tc2_destroy", _p(x), _p(wp), _p(bias), _p(out), B, H, W,
         Cin, Cout)
    _within(out, y64.detach().permute(0, 2, 3, 1), "forward")

    dx = torch.full((B, H, W, Cin), float("nan"), device=DEV)                 # every element must be written
    wt = w.reshape(Cout, Cin, 9).permute(2, 1, 0).contiguous()                 # [tap][Cin][Cout]
    _run("pdae_conv_tc2_create_s2_dgrad", "pdae_conv_tc2_run", "pdae_conv_tc2_destroy", _p(dy), _p(wt), _p(dx), B, H, W, Cin,
         Cout)
    _within(dx, x64.grad.permute(0, 2, 3, 1), "dgrad")

    dw = torch.zeros(9, Cin, Cout, device=DEV)
    _run("pdae_wgrad_tc_create_bf16_s2", "pdae_wgrad_tc_run", "pdae_wgrad_tc_destroy", _p(x), _p(dy), _p(dw), B, H, W, Cin, Cout)
    _within(dw, w64.grad.reshape(Cout, Cin, 9).permute(2, 1, 0), "wgrad")


# ---- helpers -----------------------------------------------------------------------------------------------------------
def _encoder(size):
    enc, _ = cases.model_case({"kind": "encoder", "size": size})
    return enc


def _to_train(enc):
    enc = enc.cuda().train()
    enc.precision = "fp32"
    return enc


def _enc_inputs(size, B=2):
    from pdae_b200.utils.synth import synth_images, synth_normal
    return synth_images(B, 3, size, 18), synth_normal((B, 512), 23)


def _enc_step(enc, inputs, autocast_dtype=None, enabled=True, scaler=None):
    """Encoder-only step with loss (z * r).sum(); returns (z, {name: grad}) and clears the gradients."""
    x, r = inputs
    if autocast_dtype is None:
        z = enc(x.cuda())
    else:
        with torch.autocast("cuda", dtype=autocast_dtype, enabled=enabled):
            z = enc(x.cuda())
    loss = (z * r.cuda()).sum()
    (scaler.scale(loss) if scaler is not None else loss).backward()
    grads = {k: p.grad.detach().clone() for k, p in enc.named_parameters() if p.grad is not None}
    if scaler is None:
        for p in enc.parameters():
            p.grad = None
    return z.detach(), grads


def _amp_trainer(enc):
    trs = [tr for tr in enc._train_cache.values() if tr.amp]
    assert len(trs) == 1, len(trs)
    return trs[0]


def _eligible_s2(enc):
    """The encoder's stride-2 convs after the 3-channel stem."""
    return [m for m in enc.modules() if isinstance(m, nn.Conv2d) and m.stride == (2, 2) and m.in_channels % 64 == 0]


def _check_amp_plans(tr, enc):
    assert tr.fwd.train_tc == "bf16" and tr.bwd.precision == "bf16"
    fwd_ops = [fn for fn, _ in tr.fwd.ops]
    bwd_ops = [fn for fn, _ in tr.bwd.ops]
    n = len(_eligible_s2(enc))
    assert n == (3 if enc.image_size == 64 else 4)
    assert fwd_ops.count("conv_tc2_s2") == n
    assert bwd_ops.count("wgrad_tc_bf16_s2") == n          # one stride-2 weight gradient per eligible conv
    assert bwd_ops.count("conv_tc2_s2_dgrad") == n          # ... and one data gradient (the stem needs none)
    # CUDA-core convs left: the 3-channel stem (forward + weight gradient) and the final Linear (forward, weight and data
    # gradient); nothing else
    assert [fn for fn in fwd_ops if fn in SIMT_CONV_OPS] == ["conv2d_simt", "conv2d_simt"]
    assert sorted(fn for fn in bwd_ops if fn in SIMT_CONV_OPS) == ["conv2d_dgrad_simt", "conv2d_wgrad_simt", "conv2d_wgrad_simt"]
    for fn, args in tr.fwd.ops + tr.bwd.ops:
        assert fn not in ("gn_apply_split3", "qkv_split3", "softmax_split3", "wgrad_tc"), fn
        if fn == "conv_tc2":
            assert not args[0].split3


# ---- 2. encoder step against oracle autograd ----------------------------------------------------------------------------
@pytest.mark.parametrize("size", [64, 128])
def test_encoder_step_under_bf16_autocast_matches_oracle(size):
    enc0 = _encoder(size)
    inputs = _enc_inputs(size)
    esd = {k: v.requires_grad_(True) for k, v in cases.sd_of(enc0).items()}
    z_ref = O.encoder_forward(esd, ENC_KIND[size], inputs[0])
    (z_ref * inputs[1]).sum().backward()
    enc = _to_train(enc0)
    z, grads = _enc_step(enc, inputs, torch.bfloat16)
    r = float((z.double().cpu() - z_ref.detach().double()).norm() / z_ref.detach().double().norm())
    print(f"{size}-px encoder under bf16 autocast: z rel-L2 {r:.2e}")
    assert r <= 5e-2
    _check_grads(grads, {k: v.grad for k, v in esd.items()}, f"{size}-px encoder bf16 autocast vs oracle")
    _check_amp_plans(_amp_trainer(enc), enc)


# ---- 3. the whole PDAE step -----------------------------------------------------------------------------------------------
def test_pdae_step_with_encoder_under_bf16_autocast_matches_oracle():
    """representation_learning_train_one_batch (gaussian_diffusion.py:234-255): the 64-px encoder and the ShiftUNet on the
    same 64-px images, the whole loss under autocast."""
    from pdae_b200.utils.synth import synth_images
    from tests.test_gpu_training_amp import SHIFT_CFG
    from tests.test_gpu_training_amp import _to_train as _dec_to_train
    dec0, enc0 = _shift_module(), _encoder(64)
    x0 = synth_images(2, 3, 64, 31)
    noise = torch.randn(x0.shape, generator=torch.Generator().manual_seed(3))
    dsd = {k: v.requires_grad_(k.startswith(("label_emb", "shift_"))) for k, v in cases.sd_of(dec0).items()}
    esd = {k: v.requires_grad_(True) for k, v in cases.sd_of(enc0).items()}
    D = O.DiffusionOracle(cases.DIFF)
    ref_loss = D.representation_learning_loss(lambda x: O.encoder_forward(esd, "celeba64", x),
                                              lambda x, t, z: O.shiftunet_forward(dsd, SHIFT_CFG, x, t, z), x0, T_STEPS, noise)
    ref_loss.backward()
    dec, enc = _dec_to_train(dec0), _to_train(enc0)
    gd = _gd()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss = _shift_loss(gd, dec, x0.cuda(), T_STEPS.cuda(), noise.cuda(), enc(x0.cuda()))
    loss.backward()
    loss, ref_loss = float(loss.detach()), float(ref_loss.detach())
    r = abs(loss - ref_loss) / abs(ref_loss)
    print(f"bf16 autocast PDAE step with the encoder: loss {loss:.6f} vs oracle {ref_loss:.6f} (rel {r:.2e})")
    assert r <= 1e-2
    got = {"enc." + k: p.grad for k, p in enc.named_parameters()}
    got.update({"dec." + k: p.grad for k, p in dec.named_parameters() if p.grad is not None})
    ref = {"enc." + k: v.grad for k, v in esd.items()}
    ref.update({"dec." + k: v.grad for k, v in dsd.items() if v.grad is not None})
    _check_grads(got, ref, "PDAE step (encoder + ShiftUNet) bf16 autocast vs oracle")
    _check_amp_plans(_amp_trainer(enc), enc)


# ---- 4. + 5. plans, fp16 autocast, GradScaler, alternation ---------------------------------------------------------------
def test_fp16_autocast_and_grad_scaler_use_the_bf16_encoder_plans():
    enc = _to_train(_encoder(64))
    inputs = _enc_inputs(64)
    z_b, g_b = _enc_step(enc, inputs, torch.bfloat16)
    tr = _amp_trainer(enc)
    z_h, g_h = _enc_step(enc, inputs, torch.float16)
    assert _amp_trainer(enc) is tr and len(enc._train_cache) == 1       # either autocast dtype: the same bf16 trainer
    assert float((z_h - z_b).norm() / z_b.norm()) <= AMP_SPREAD["rel"]
    _check_grads(g_h, g_b, "fp16 vs bf16 autocast encoder", **AMP_SPREAD)
    # the reference trainer's sequence: scaler.scale(loss).backward(); scaler.step(opt); scaler.update()
    scaler = torch.amp.GradScaler("cuda")
    opt = torch.optim.Adam(list(enc.parameters()), lr=1e-4)
    _, g_s = _enc_step(enc, inputs, torch.float16, scaler=scaler)
    scale = float(scaler.get_scale())
    assert _amp_trainer(enc) is tr and scale > 1
    assert all(torch.isfinite(g).all() for g in g_s.values())
    _check_grads({k: g / scale for k, g in g_s.items()}, g_b, f"GradScaler (scale {scale:g}) grads / scale vs unscaled",
                 **AMP_SPREAD)
    before = [p.detach().clone() for p in enc.parameters()]
    scaler.step(opt)
    scaler.update()
    assert any(not torch.equal(p, q) for p, q in zip(enc.parameters(), before)), "GradScaler skipped a finite step"


def test_alternating_amp_and_full_precision_encoder_steps():
    enc = _to_train(_encoder(64))
    fresh = copy.deepcopy(enc)            # never sees autocast
    inputs = _enc_inputs(64)
    z_ref, g_ref = _enc_step(fresh, inputs)
    z_amp1, g_amp1 = _enc_step(enc, inputs, torch.bfloat16)
    z_full, g_full = _enc_step(enc, inputs)
    z_amp2, g_amp2 = _enc_step(enc, inputs, torch.bfloat16)
    assert len(enc._train_cache) == 2     # one full-precision and one AMP trainer, each with its own buffers
    full_tr = [tr for tr in enc._train_cache.values() if not tr.amp][0]
    z_off, g_off = _enc_step(enc, inputs, torch.bfloat16, enabled=False)
    assert len(enc._train_cache) == 2 and [tr for tr in enc._train_cache.values() if not tr.amp][0] is full_tr
    fresh_tr = list(fresh._train_cache.values())[0]
    assert not fresh_tr.amp and fresh_tr.fwd.train_tc is None
    # the full-precision trainer of the encoder that saw autocast records exactly the plans of one that never did
    for a, b in ((full_tr.fwd, fresh_tr.fwd), (full_tr.bwd, fresh_tr.bwd)):
        assert a.precision == b.precision and a.train_tc == b.train_tc
        assert [(fn, [(x.shape, x.dtype) if hasattr(x, "shape") else None for x in args]) for fn, args in a.ops] == \
               [(fn, [(x.shape, x.dtype) if hasattr(x, "shape") else None for x in args]) for fn, args in b.ops]
    assert sum(fn == "conv2d_wgrad_simt" for fn, _ in full_tr.bwd.ops) == 1 + len(_eligible_s2(enc)) + 1
    for z, what in ((z_full, "full precision after AMP"), (z_off, "autocast(enabled=False)")):
        assert float((z - z_ref).norm() / z_ref.norm()) <= FP32_SPREAD["rel"], what
    _check_grads(g_full, g_ref, "full precision after AMP vs never-autocast encoder", **FP32_SPREAD)
    _check_grads(g_off, g_ref, "autocast(enabled=False) vs never-autocast encoder", **FP32_SPREAD)
    assert float((z_amp2 - z_amp1).norm() / z_amp1.norm()) <= AMP_SPREAD["rel"]
    _check_grads(g_amp2, g_amp1, "AMP step after a full-precision step vs the first", **AMP_SPREAD)
