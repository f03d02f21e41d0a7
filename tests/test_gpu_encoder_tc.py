"""The semantic encoder's forward on the tensor cores in the "bf16" and "bf16x3" modes: the stride-2 forward with a bf16 output
and GroupNorm statistics, its split-operand form, the stride-2 stem and the split-operand final Linear through the C-ABI
against float64; the whole encoder against the CPU oracle with the plans it records; packed-weight refresh; the callers that
run a frozen encoder (latent DPM training, manipulation training, autoencoding)."""
import ctypes

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import pdae_oracle as O
from pdae_b200 import _native
from pdae_b200._native import PDAE_BF16, PDAE_F32, RESAMPLE_NONE
from pdae_b200.engine import split3_weights
from tests import cases
from tests.test_gpu_encoder_amp import ENC_KIND, S2_SHAPES
from tests.test_gpu_parity import check
from tests.util import assert_close, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"
# B = 3 and B = 129 leave a partial multi-image tile at the 8x8 and 4x4 output grids
S2_CASES = [(B,) + s for s in S2_SHAPES for B in (2, 3, 32, 129)]


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _run_tc2(create, *args):
    L = _native.lib()
    h = ctypes.c_void_p()
    _native.check(getattr(L, create)(ctypes.byref(h), *args), create)
    try:
        _native.check(L.pdae_conv_tc2_run(h, _stream()), "pdae_conv_tc2_run")
        torch.cuda.synchronize()
    finally:
        L.pdae_conv_tc2_destroy(h)


def _split3(x):
    """[..., C] fp32 -> [..., 3 C] bf16 = [hi | lo | hi] by the library's own splitting kernel (gn_apply_split3, identity affine)."""
    B, H, W, C = x.shape
    out = torch.empty(B, H, W, 3 * C, device=DEV, dtype=torch.bfloat16)
    _native.check(_native.lib().pdae_gn_apply_split3(_p(x), C, None, 0, None, 0, RESAMPLE_NONE, B, H, W, _p(out), None, PDAE_F32,
                                                     _stream()), "pdae_gn_apply_split3")
    return out


def _bf16_ulp(v):
    _, e = torch.frexp(v)
    return torch.ldexp(torch.ones_like(v), e - 8)     # |v| in [2^(e-1), 2^e): bf16 spacing 2^(e-1-7)


def _within_bf16(got, ref, what):
    """Every element within one bf16 ulp of the float64 value plus 2e-5 of max|ref|."""
    scale = ref.abs().max().item()
    err = (got.double() - ref).abs()
    bound = _bf16_ulp(ref) + 2e-5 * scale
    worst = (err / bound).max().item()
    print(f"{what}: max|err| {err.max().item():.3e}, worst err / (ulp + 2e-5 max|ref|) {worst:.3f}")
    assert torch.isfinite(got.float()).all(), f"{what}: non-finite output (an element not written?)"
    assert worst <= 1.0, (what, worst)


def _within(got, ref, what, tol=2e-5):
    scale = ref.abs().max().item()
    err = (got.double() - ref).abs().max().item()
    print(f"{what}: max|err| {err:.3e} = {err / scale:.2e} of max|ref| {scale:.3e}")
    assert torch.isfinite(got).all(), f"{what}: non-finite output (an element not written?)"
    assert err <= tol * scale, (what, err, scale)


def _check_stats(stats, out, what):
    """ch_stats [B][C][2] against float64 sums of the stored values over each image: relative to the sum of |v| (sum) and to the
    sum itself (sum of squares) per channel, <= 1e-4."""
    v = out.double().flatten(1, 2)                                  # [B][HW][C]
    s, q, a = v.sum(1), (v * v).sum(1), v.abs().sum(1)
    es = ((stats[..., 0].double() - s).abs() / a.clamp_min(1e-30)).max().item()
    eq = ((stats[..., 1].double() - q).abs() / q.clamp_min(1e-30)).max().item()
    print(f"{what}: statistics rel err sum {es:.2e}, sum^2 {eq:.2e}")
    assert es <= 1e-4 and eq <= 1e-4, (what, es, eq)


def _case(B, H, Cin, Cout, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = (torch.randn(B, H, H, Cin, generator=g) * 1.3 + 0.2).to(DEV)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (3 * Cin ** 0.5)).to(DEV)
    bias = (torch.randn(Cout, generator=g) * 0.5).to(DEV)
    return x, w, bias


def _conv64(x, w, bias):
    return F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), bias.double(), stride=2, padding=1).permute(0, 2, 3, 1)


# ---- 1. stride-2 forward: bf16 / fp32 output and statistics ----------------------------------------------------------------
@pytest.mark.parametrize("B,H,Cin,Cout", S2_CASES)
def test_stride2_forward_bf16_output_and_statistics(B, H, Cin, Cout):
    x, w, bias = _case(B, H, Cin, Cout, H * 7 + Cin + B)
    xb, wb = x.to(torch.bfloat16).contiguous(), w.to(torch.bfloat16)
    ref = _conv64(xb, wb, bias)                      # the products of bf16 values are exact; only the summation differs
    wp = wb.reshape(Cout, Cin, 9).permute(2, 0, 1).contiguous()
    for dt, odt in ((torch.float32, PDAE_F32), (torch.bfloat16, PDAE_BF16)):
        out = torch.full((B, H // 2, H // 2, Cout), float("nan"), device=DEV, dtype=dt)
        stats = torch.zeros(B, Cout, 2, device=DEV)
        _run_tc2("pdae_conv_tc2_create_s2_ex", _p(xb), _p(wp), _p(bias), _p(out), odt, _p(stats), B, H, H, Cin, Cout)
        what = f"B={B} {H}x{H} {Cin}->{Cout} {str(dt)[6:]}"
        if dt == torch.float32:
            _within(out, ref, what)
        else:
            _within_bf16(out, ref, what)
        _check_stats(stats, out, what)


# ---- 2. the split-operand stride-2 forward (fp32-grade) ---------------------------------------------------------------------
@pytest.mark.parametrize("B,H,Cin,Cout", S2_CASES)
def test_split_operand_stride2_forward_is_fp32_grade(B, H, Cin, Cout):
    x, w, bias = _case(B, H, Cin, Cout, H * 11 + Cin + B)
    ref = _conv64(x, w, bias)                        # float64 conv of the unrounded fp32 operands
    x3 = _split3(x.contiguous())
    w3 = split3_weights(w.reshape(Cout, Cin, 9))     # [9][Cout][W_hi | W_hi | W_lo]
    out = torch.full((B, H // 2, H // 2, Cout), float("nan"), device=DEV)
    stats = torch.zeros(B, Cout, 2, device=DEV)
    _run_tc2("pdae_conv_tc2_create_s2_ex", _p(x3), _p(w3), _p(bias), _p(out), PDAE_F32, _p(stats), B, H, H, 3 * Cin, Cout)
    assert torch.isfinite(out).all()
    r = rel_l2(out, ref)
    m = ((out.double() - ref).abs().max() / ref.abs().max()).item()
    print(f"split-operand B={B} {H}x{H} {Cin}->{Cout}: rel-L2 {r:.2e}, max|err| {m:.2e} of max|ref|")
    assert r <= 5e-5 and m <= 1e-4, (r, m)
    _check_stats(stats, out, "split-operand")


# ---- 3. stride-2 stem and split-operand Linear ----------------------------------------------------------------------------
@pytest.mark.parametrize("size,B", [(64, 2), (64, 33), (128, 2), (128, 16)])
def test_stride2_stem_matches_float64(size, B):
    g = torch.Generator(device="cpu").manual_seed(size + B)
    x = torch.randn(B, 3, size, size, generator=g).clamp(-1, 1).to(DEV)
    w = (torch.randn(64, 3, 3, 3, generator=g) * 0.2).to(DEV)
    bias = (torch.randn(64, generator=g) * 0.1).to(DEV)
    ref = F.conv2d(x.double(), w.double(), bias.double(), stride=2, padding=1).permute(0, 2, 3, 1)
    wp = w.reshape(64, 3, 9).permute(2, 1, 0).contiguous()                      # [9][Cin][Cout]
    out = torch.full((B, size // 2, size // 2, 64), float("nan"), device=DEV, dtype=torch.bfloat16)
    stats = torch.zeros(B, 64, 2, device=DEV)
    _native.check(_native.lib().pdae_stem_conv_s2_bf16(_p(x), _p(wp), _p(bias), _p(out), _p(stats), B, size, size, 3, 64,
                                                       _stream()), "pdae_stem_conv_s2_bf16")
    torch.cuda.synchronize()
    _within_bf16(out, ref, f"stem {size} px B={B}")
    _check_stats(stats, out, f"stem {size} px B={B}")


@pytest.mark.parametrize("size,B", [(64, 2), (64, 128), (128, 2), (128, 128)])
def test_split_operand_final_linear_matches_float64(size, B):
    """The encoder's View(-1, C*4*4) + Linear on a split activation: K = 3 HW C (12288 for the 128-px encoder) on the split-K
    GEMM, the weight packed per pixel as [W_hi | W_hi | W_lo] in NHWC-flatten order."""
    C, D, HW = (128 if size == 64 else 256), 512, 16
    g = torch.Generator(device="cpu").manual_seed(size * 3 + B)
    act = torch.randn(B, 4, 4, C, generator=g).to(DEV)                           # NHWC
    wt = (torch.randn(D, C * HW, generator=g) / (C * HW) ** 0.5).to(DEV)        # reference: NCHW flatten (c, y, x)
    bias = (torch.randn(D, generator=g) * 0.1).to(DEV)
    ref = F.linear(act.double().permute(0, 3, 1, 2).reshape(B, -1), wt.double(), bias.double())
    w = wt.reshape(D, C, HW).permute(0, 2, 1)
    hi = w.to(torch.bfloat16)
    wp = torch.cat([hi, hi, (w - hi.float()).to(torch.bfloat16)], dim=2).reshape(D, 3 * HW * C).contiguous()
    a3 = _split3(act.contiguous())
    out = torch.zeros(B, D, device=DEV)
    _run_tc2("pdae_conv_tc2_create_splitk", _p(a3), _p(wp), _p(bias), _p(out), B, 3 * HW * C, D)
    r = rel_l2(out, ref)
    m = ((out.double() - ref).abs().max() / ref.abs().max()).item()
    print(f"split-operand Linear {size} px B={B} K={3 * HW * C}: rel-L2 {r:.2e}, max|err| {m:.2e} of max|ref|")
    assert r <= 5e-5 and m <= 1e-4, (r, m)


# ---- 4. the whole encoder against the oracle, and its plans -----------------------------------------------------------------
def _encoder(size):
    enc, _ = cases.model_case({"kind": "encoder", "size": size})
    return enc


def _eligible_s2(enc):
    """The encoder's stride-2 convs after the 3-channel stem."""
    return [m for m in enc.modules() if isinstance(m, nn.Conv2d) and m.stride == (2, 2) and m.in_channels % 64 == 0]


def _plan(enc, precision):
    ents = [v for k, v in enc._plans().items() if k[1] == precision]
    assert len(ents) == 1
    return ents[0][0]


def _check_plan(plan, enc, precision):
    ops = [fn for fn, _ in plan.ops]
    n = len(_eligible_s2(enc))
    if precision == "fp32":
        assert not any(fn.startswith(("conv_tc", "gemm_tc", "stem_")) for fn in ops), ops
        assert ops.count("conv2d_simt") >= 2 + n
        return
    assert ops.count("conv_tc2_s2") == n
    assert ops.count("conv2d_simt") == (0 if precision == "bf16" else 1)   # bf16x3: the fp32-grade CUDA-core stem
    assert ("stem_conv_s2_bf16" in ops) == (precision == "bf16")
    first_tc = ops.index("conv_tc2_s2")
    assert all(i < first_tc for i, fn in enumerate(ops) if fn == "ch_stats"), "ch_stats after a tensor-core conv"
    assert ops.count("ch_stats") == (0 if precision == "bf16" else 1)
    assert "conv_tc2_splitk" in ops                                          # the final Linear
    for fn, args in plan.ops:
        if fn == "conv_tc2_s2":
            assert bool(args[0].split3) == (precision == "bf16x3")
            assert args[3].dtype == (torch.bfloat16 if precision == "bf16" else torch.float32)
            assert args[5] is not None                                      # the epilogue feeds the next GroupNorm


@pytest.mark.parametrize("B", [2, 16])
@pytest.mark.parametrize("size", [64, 128])
def test_encoder_matches_oracle_in_tensor_core_modes(size, B):
    from pdae_b200.utils.synth import synth_images
    enc = _encoder(size)
    x = synth_images(B, 3, size, 18)
    with torch.no_grad():
        ref = O.encoder_forward(cases.sd_of(enc), ENC_KIND[size], x)
    enc = enc.cuda()
    for precision in ("bf16x3", "bf16", "fp32"):
        enc.precision = precision
        with torch.no_grad():
            z = enc(x.cuda())
        check(z, ref, precision, f"{size}-px encoder B={B}")
        _check_plan(_plan(enc, precision), enc, precision)


# ---- 5. packed weights follow the parameters --------------------------------------------------------------------------------
def _same(got, want, precision, what):
    """Two runs of one plan.  The GroupNorm statistics are accumulated with atomics, so their last bits vary from run to run.
    In "bf16x3" that stays at the fp32 level.  In "bf16" such a bit can move a value across a bf16 rounding boundary of the
    normalised activation, and the deep stack carries it to z (up to about 1e-2 of |z| ~ 1 on the 128-px encoder at B = 4):
    the mode's stated tolerance applies."""
    print(f"[{precision}] {what}: rel-L2 {rel_l2(got, want):.2e}")
    if precision == "bf16x3":
        assert_close(got, want, what=what, rtol=1e-3, atol=1e-4)
    else:
        check(got, want, precision, what)


def _perturb(p):
    """A smooth per-element factor in [0.8, 1.2]: unlike a uniform scale, GroupNorm does not cancel it."""
    return p * (1.0 + 0.2 * torch.sin(torch.arange(p.numel(), device=p.device, dtype=p.dtype).reshape(p.shape)))


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_encoder_packed_weights_refresh(precision):
    from pdae_b200.utils.synth import synth_images
    enc = _encoder(128).cuda()
    enc.precision = precision
    x = synth_images(4, 3, 128, 19).cuda()
    with torch.no_grad():
        z1 = enc(x)
        _same(enc(x), z1, precision, "repeat call")
        sd = {k: v.clone() for k, v in enc.state_dict().items()}
        for p in enc.parameters():               # versioned in-place update: every packed copy must be re-derived
            p.copy_(_perturb(p))
        z2 = enc(x)
        assert rel_l2(z2, z1) > 1e-1, "stale packed weights: output did not change"
        check(z2, O.encoder_forward(cases.sd_of(enc), "ffhq128", x.cpu()), precision, "perturbed weights vs oracle")
        enc.load_state_dict(sd)
        _same(enc(x), z1, precision, "load_state_dict restores")
        for p in enc.parameters():               # a write that bumps no version counter, then invalidate_packed()
            p.data.copy_(_perturb(p.data))
        enc.invalidate_packed()
        _same(enc(x), z2, precision, "invalidate_packed after .data writes")
    assert len(enc._plans()) == 1


# ---- 6. callers of the frozen encoder ---------------------------------------------------------------------------------------
def _frozen(size, precision):
    enc = _encoder(size).cuda().requires_grad_(False).eval()
    enc.precision = precision
    return enc


class _Recorder:
    """Calls the encoder and keeps what it returned (z is consumed inside the caller)."""

    def __init__(self, enc):
        self.enc, self.z = enc, []

    def __call__(self, x):
        z = self.enc(x)
        self.z.append(z.detach().clone())
        return z


def _stats():
    from pdae_b200.utils.synth import synth_normal
    return (synth_normal((1, 512), 34) * 0.1).cuda(), (synth_normal((1, 512), 35).abs() + 0.5).cuda()


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_latent_diffusion_and_manipulation_training_with_tensor_core_encoder(precision):
    from pdae_b200.utils.synth import synth_images, synth_normal
    from tests.test_gpu_latent_amp import _ffhq_setup, _gd
    mean, std = _stats()
    x0 = synth_images(16, 3, 64, 33).cuda()
    with torch.no_grad():
        z_fp32 = _frozen(64, "fp32")(x0)
    enc = _Recorder(_frozen(64, precision))
    gd = _gd()
    _, mlp, _, _ = _ffhq_setup(dropout=0.1, B=16)
    mlp = mlp.cuda().train()
    for amp in (False, True):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            loss = gd.latent_diffusion_train_one_batch(mlp, enc, x0, mean, std)["prediction_loss"]
        loss.backward()
        assert torch.isfinite(loss), (precision, amp)
        assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in mlp.parameters()), (precision, amp)
        mlp.zero_grad(set_to_none=True)
    classifier = nn.Linear(512, 40).cuda()
    label = torch.where(synth_normal((16, 40), 36) > 0, 1.0, -1.0).cuda()
    loss = gd.manipulation_train_one_batch(classifier, enc, x0, label, mean, std)["bce_loss"]
    loss.backward()
    assert torch.isfinite(loss) and all(torch.isfinite(p.grad).all() for p in classifier.parameters())
    assert len(enc.z) == 3
    for z in enc.z:
        check(z, z_fp32, precision, f"frozen {precision} encoder z vs the fp32-mode encoder")


def test_autoencoding_with_split_operand_encoder_matches_fp32_recon_mse():
    from pdae_b200.utils.synth import synth_images
    from tests.test_gpu_diffusion import gd
    from tests.util import load_golden
    cfg, _ = load_golden("loop_autoencode_ddim10")
    dec, _ = cases.model_case({"kind": "shiftunet", "cfg": cfg["cfg"], "size": 64})
    dec = dec.cuda()
    dec.precision = "fp32"
    enc = _encoder(64).cuda()
    x0 = synth_images(2, 3, 64, 28).cuda()
    mse = lambda a, b: float((((a.cpu() + 1) / 2 - (b.cpu() + 1) / 2) ** 2).mean())
    res = {}
    for precision in ("fp32", "bf16x3"):
        enc.precision = precision
        with torch.no_grad():
            res[precision] = mse(gd().representation_learning_autoencoding("ddim10", "ddim10", enc, dec, x0), x0)
    d = abs(res["bf16x3"] - res["fp32"])
    print(f"recon MSE: fp32-mode encoder {res['fp32']:.6e}, bf16x3 encoder {res['bf16x3']:.6e}, delta {d:.3e}")
    assert d <= 1e-5
