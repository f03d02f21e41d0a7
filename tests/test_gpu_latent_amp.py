"""Latent-DPM training under torch.autocast (the reference's enable_amp in trainer/train_latent_diffusion.py): the split-K
Linear GEMM and the fused bf16 modulate / LayerNorm / SiLU / dropout kernels through the C-ABI, the bf16 MLPSkipNet
training step against oracle autograd on the CPU, the plans it records, and how callers use it (fp16 autocast,
GradScaler, AMP and full-precision steps on one module, the full latent_diffusion_train_one_batch call)."""
import copy
import ctypes

import pytest
import torch

from oracle import pdae_oracle as O
from pdae_b200 import _native
from tests import cases
from tests.configs import FFHQ_LATENT
from tests.test_gpu_training import _latent_loss, _latent_setup
from tests.test_gpu_training_amp import AMP_SPREAD, FP32_SPREAD, SPLIT_OPS, _check_grads
from tests.util import load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16_OPS = ("conv_tc2_splitk", "mlp_mod_ln_act_bf16", "mlp_mod_ln_act_bwd_bf16", "copy_cols_bf16")


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- 1. split-K GEMM ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,K,N", [(3, 512, 256), (128, 2560, 2048), (128, 2560, 512), (200, 2560, 2048), (128, 18432, 512),
                                   (128, 512, 18432)])
def test_splitk_linear_matches_float64_matmul_of_rounded_operands(B, K, N):
    g = torch.Generator(device="cpu").manual_seed(B + K + N)
    x = (torch.randn(B, K, generator=g) * 0.7).to(DEV).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).to(DEV).to(torch.bfloat16)
    bias = torch.randn(N, generator=g).to(DEV)
    out = torch.full((B, N), float("nan"), device=DEV)
    L = _native.lib()
    h = ctypes.c_void_p()
    _native.check(L.pdae_conv_tc2_create_splitk(ctypes.byref(h), _p(x), _p(w), _p(bias), _p(out), B, K, N),
                  "pdae_conv_tc2_create_splitk")
    try:
        for _ in range(2):     # the output is zeroed before every run, as the plan's pdae_zero op does
            out.zero_()
            _native.check(L.pdae_conv_tc2_run(h, _st()), "pdae_conv_tc2_run")
        torch.cuda.synchronize()
    finally:
        L.pdae_conv_tc2_destroy(h)
    ref = x.double() @ w.double().t() + bias.double()
    scale = float(ref.abs().max())
    err = float((out.double() - ref).abs().max())
    print(f"split-K B={B} K={K} N={N}: max err / max|ref| = {err / scale:.2e}")
    assert err <= 2e-5 * scale, (err, scale)


# ---- 2. fused kernels --------------------------------------------------------------------------------------------------
def _rows(B, N, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(B, N, generator=g) * scale).to(DEV)


@pytest.mark.parametrize("ln", [True, False])
@pytest.mark.parametrize("masked", [True, False])
@pytest.mark.parametrize("cond_ld", [0, 256, 1024])     # 0: no cond; 1024: the cond block sits at column 256 of [B][1024]
def test_fused_forward_bf16_is_the_rounding_of_the_fp32_kernels(ln, masked, cond_ld):
    B, N, D = 7, 256, 128
    L = _native.lib()
    h = _rows(B, N, 1, 2.0)
    bank = _rows(B, cond_ld, 2, 0.5) if cond_ld else None
    off = 256 if cond_ld > N else 0
    cond_c = bank[:, off:off + N].contiguous() if cond_ld else None       # what the fp32 kernel reads
    lw, lb = (_rows(1, N, 3).flatten() + 1, _rows(1, N, 4).flatten()) if ln else (None, None)
    mask = (torch.rand(B, N, generator=torch.Generator().manual_seed(5)) > 0.1).float().to(DEV) if masked else None
    scale = 1.0 / 0.9
    ref = torch.zeros(B, N + D, device=DEV)
    _native.check(L.pdae_mlp_mod_ln_act(_p(h), _p(cond_c), _p(lw), _p(lb), ctypes.c_float(1e-5), 1, _p(ref), N + D, B, N,
                                        _st()), "mlp_mod_ln_act")
    if masked:
        _native.check(L.pdae_mul_mask_cols(_p(ref), N + D, _p(mask), ctypes.c_float(scale), B, N, _st()), "mul_mask_cols")
    got = torch.zeros(B, N + D, device=DEV, dtype=torch.bfloat16)
    cptr = ctypes.c_void_p(bank[:, off:].data_ptr()) if cond_ld else None
    _native.check(L.pdae_mlp_mod_ln_act_bf16(_p(h), cptr, cond_ld, _p(lw), _p(lb), ctypes.c_float(1e-5), 1, _p(mask),
                                             ctypes.c_float(scale), _p(got), N + D, B, N, _st()), "mlp_mod_ln_act_bf16")
    z = _rows(B, D, 6)
    _native.check(L.pdae_copy_cols_bf16(_p(z), _p(got), N + D, N, B, D, _st()), "copy_cols_bf16")
    torch.cuda.synchronize()
    assert torch.equal(got[:, :N], ref[:, :N].to(torch.bfloat16))
    assert torch.equal(got[:, N:], z.to(torch.bfloat16))


@pytest.mark.parametrize("ln", [True, False])
@pytest.mark.parametrize("masked", [True, False])
def test_fused_backward_matches_fp32_kernel_bitwise_and_rounds_it(ln, masked):
    B, N, ld, off, dy_ld = 5, 256, 768, 256, 320
    L = _native.lib()
    h = _rows(B, N, 11, 2.0)
    bank = _rows(B, ld, 12, 0.5)
    cond = bank[:, off:]
    dy = _rows(B, dy_ld, 13)
    lw, lb = (_rows(1, N, 14).flatten() + 1, _rows(1, N, 15).flatten()) if ln else (None, None)
    mask = (torch.rand(B, N, generator=torch.Generator().manual_seed(16)) > 0.1).float().to(DEV) if masked else None
    scale = 1.0 / 0.9
    # fp32 reference: mask applied in place on dy, then the fp32 backward on a contiguous cond
    dy_ref = dy.clone()
    if masked:
        _native.check(L.pdae_mul_mask_cols(_p(dy_ref), dy_ld, _p(mask), ctypes.c_float(scale), B, N, _st()), "mul_mask_cols")
    dh_ref, dc_ref = torch.empty(B, N, device=DEV), torch.empty(B, N, device=DEV)
    dlw_ref, dlb_ref = (torch.zeros(N, device=DEV), torch.zeros(N, device=DEV)) if ln else (None, None)
    _native.check(L.pdae_mlp_mod_ln_act_bwd(_p(h), _p(cond[:, :N].contiguous()), _p(lw), _p(lb), ctypes.c_float(1e-5), 1,
                                            _p(dy_ref), dy_ld, _p(dh_ref), _p(dc_ref), _p(dlw_ref), _p(dlb_ref), B, N, _st()),
                  "mlp_mod_ln_act_bwd")
    dh, dh_bf = torch.empty(B, N, device=DEV), torch.empty(B, N, device=DEV, dtype=torch.bfloat16)
    dbank = torch.zeros(B, ld, device=DEV)
    dbank_bf = torch.zeros(B, ld, device=DEV, dtype=torch.bfloat16)
    dlw, dlb = (torch.zeros(N, device=DEV), torch.zeros(N, device=DEV)) if ln else (None, None)
    _native.check(L.pdae_mlp_mod_ln_act_bwd_bf16(_p(h), ctypes.c_void_p(cond.data_ptr()), ld, _p(lw), _p(lb),
                                                 ctypes.c_float(1e-5), 1, _p(dy), dy_ld, _p(mask), ctypes.c_float(scale), _p(dh),
                                                 _p(dh_bf), ctypes.c_void_p(dbank[:, off:].data_ptr()),
                                                 ctypes.c_void_p(dbank_bf[:, off:].data_ptr()), _p(dlw), _p(dlb), B, N, _st()),
                  "mlp_mod_ln_act_bwd_bf16")
    torch.cuda.synchronize()
    dc = dbank[:, off:off + N]
    assert torch.equal(dh, dh_ref) and torch.equal(dc, dc_ref)
    assert torch.equal(dh_bf, dh.to(torch.bfloat16)) and torch.equal(dbank_bf[:, off:off + N], dc.to(torch.bfloat16))
    assert not dbank[:, :off].any() and not dbank[:, off + N:].any()        # only its own column block is written
    if ln:   # (sums of fp32 atomics over the rows: equal up to the order of the additions)
        torch.testing.assert_close(dlw, dlw_ref, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(dlb, dlb_ref, rtol=1e-5, atol=1e-6)


# ---- 3. the latent step under bf16 autocast ----------------------------------------------------------------------------
def _gd():
    from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
    return GaussianDiffusion(cases.DIFF, torch.device(DEV))


def _ffhq_setup(dropout=0.0, B=128):
    from pdae_b200.model.mlp_skip_net import MLPSkipNet
    from pdae_b200.utils.synth import fill_module_, synth_normal
    c = dict({k: v for k, v in FFHQ_LATENT.items() if k != "model"}, dropout=dropout)
    mlp = fill_module_(MLPSkipNet(**c), seed=79)
    sd = {k: v.requires_grad_(True) for k, v in cases.sd_of(mlp).items() if ".cond_layers." not in k}
    g = {"z0": synth_normal((B, c["input_channel"]), 81), "noise": synth_normal((B, c["input_channel"]), 82),
         "t": torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(83))}
    return c, mlp, sd, g


def _fixture_setup(dropout=0.0):
    cfg, g = load_golden("train_latent")
    c, mlp, sd = _latent_setup(cfg, dropout=dropout)
    return c, mlp, sd, g


def _step(gd, mlp, g, autocast_dtype=torch.bfloat16, enabled=True):
    with torch.autocast("cuda", dtype=autocast_dtype or torch.bfloat16, enabled=enabled and autocast_dtype is not None):
        loss = _latent_loss(gd, mlp, g["z0"].cuda(), g["t"].cuda(), g["noise"].cuda())
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in mlp.named_parameters()}
    for p in mlp.parameters():
        p.grad = None
    return loss.detach(), grads


def _amp_trainer(mlp):
    trs = [tr for tr in mlp._train_cache.values() if tr.amp]
    assert len(trs) == 1, len(trs)
    return trs[0]


def _check_amp_plans(tr, n_layers):
    fwd_ops = [fn for fn, _ in tr.fwd.ops]
    n_gemm = fwd_ops.count("conv_tc2") + fwd_ops.count("conv_tc2_splitk")
    assert n_gemm == n_layers + 1, fwd_ops          # every layer's Linear + ONE bank GEMM for all linear_emb
    assert fwd_ops.count("conv2d_simt") == 2        # time_embed only
    assert fwd_ops.count("mlp_mod_ln_act_bf16") == n_layers          # the bank operand + each conditioned layer
    bwd_ops = [fn for fn, _ in tr.bwd.ops]
    assert not set(bwd_ops) & set(SPLIT_OPS), bwd_ops
    assert bwd_ops.count("wgrad_tc_bf16") >= n_layers + 1
    assert bwd_ops.count("mlp_mod_ln_act_bwd_bf16") == n_layers - 1 and "add_inplace" not in bwd_ops
    assert "conv_tc2_splitk" in bwd_ops


@pytest.mark.parametrize("which", ["fixture", "ffhq_latent"])
@pytest.mark.parametrize("dropout", [0.0, 0.1])
def test_latent_step_under_bf16_autocast_matches_oracle(which, dropout):
    """The L1 loss's gradient w.r.t. the prediction is sign(prediction - noise) / N.  bf16 forward operands move a few
    predictions across their target (44 of 65536 on the ffhq_latent net), and those flipped signs alone move the linear
    weights' gradients by ~5e-2 rel-L2 (float64 emulation of the same roundings: 5.2e-2 with the oracle's signs, 1.0e-2 with
    the bf16 step's own).  So the loss is checked against the oracle's, and the gradients against oracle autograd of the same
    L1 loss with the bf16 step's signs: that isolates the trainer's own arithmetic."""
    c, mlp, sd, g = (_fixture_setup if which == "fixture" else _ffhq_setup)(dropout)
    mlp = mlp.cuda().train()
    gd = _gd()
    torch.manual_seed(3)
    lc = gd.latent_diffusion_config
    with torch.autocast("cuda", dtype=torch.bfloat16):
        z0, t, noise = g["z0"].cuda(), g["t"].cuda(), g["noise"].cuda()
        z_t = gd.extract_coef_at_t(lc["sqrt_alphas_cumprod"], t, z0.shape) * z0 + \
            gd.extract_coef_at_t(lc["sqrt_one_minus_alphas_cumprod"], t, z0.shape) * noise
        pred = mlp(z_t, t)
        loss = gd.p_loss(noise, pred, loss_type=lc["loss_type"])
    loss.backward()
    loss = loss.detach()
    grads = {k: p.grad for k, p in mlp.named_parameters()}
    sign = torch.sign(pred.detach().cpu() - g["noise"])
    tr = _amp_trainer(mlp)
    if dropout:
        names = {id(m): n for n, m in mlp.named_modules()}
        masks = {names[id(layer)]: mk.tensor.cpu().clone() for layer, mk, p in tr.fwd.dropout_masks}
        assert len(masks) == c["num_layers"] - 1
        O.DROPOUT_MASKS = dict(masks, p=dropout)
    pred_ref = {}

    def fn(z, tt):
        pred_ref["y"] = O.mlp_skip_net_forward(sd, c, z, tt)
        return pred_ref["y"]
    try:
        ref = O.DiffusionOracle(cases.DIFF).latent_diffusion_loss(fn, g["z0"], g["t"], g["noise"])
        (sign * (pred_ref["y"] - g["noise"])).mean().backward()
    finally:
        O.DROPOUT_MASKS = None
    ref = ref.detach()
    flips = int((sign != torch.sign(pred_ref["y"].detach() - g["noise"])).sum())
    r = abs(float(loss) - float(ref)) / abs(float(ref))
    print(f"{which} dropout={dropout}: loss {float(loss):.6f} vs oracle {float(ref):.6f} (rel {r:.2e}); "
          f"{flips} of {sign.numel()} L1 signs differ")
    assert r <= 1e-2 and flips <= 1e-3 * sign.numel()
    _check_grads(grads, {k: v.grad for k, v in sd.items()}, f"latent {which} bf16 autocast vs oracle")
    _check_amp_plans(tr, c["num_layers"])


# ---- 4. plans of the full-precision trainer; 5. callers ----------------------------------------------------------------
def test_full_precision_trainer_is_unchanged_and_alternates_with_amp():
    c, mlp, sd, g = _fixture_setup()
    mlp = mlp.cuda().train()
    fresh = copy.deepcopy(mlp)                       # never sees autocast
    gd = _gd()
    _, g_ref = _step(gd, fresh, g, None)
    _, g_amp1 = _step(gd, mlp, g)
    _, g_full = _step(gd, mlp, g, None)
    _, g_amp2 = _step(gd, mlp, g)
    assert len(mlp._train_cache) == 2
    full_tr = [tr for tr in mlp._train_cache.values() if not tr.amp][0]
    _, g_off = _step(gd, mlp, g, torch.bfloat16, enabled=False)
    assert len(mlp._train_cache) == 2 and [tr for tr in mlp._train_cache.values() if not tr.amp][0] is full_tr
    fresh_tr = list(fresh._train_cache.values())[0]
    for a, b in ((full_tr.fwd, fresh_tr.fwd), (full_tr.bwd, fresh_tr.bwd)):
        assert a.precision == b.precision
        ops_a = [(fn, [(x.shape, x.dtype) if hasattr(x, "shape") else None for x in args]) for fn, args in a.ops]
        ops_b = [(fn, [(x.shape, x.dtype) if hasattr(x, "shape") else None for x in args]) for fn, args in b.ops]
        assert ops_a == ops_b
        assert not {fn for fn, _ in a.ops} & set(BF16_OPS)
    _check_grads(g_full, g_ref, "full precision after AMP vs never-autocast module", **FP32_SPREAD)
    _check_grads(g_off, g_ref, "autocast(enabled=False) vs never-autocast module", **FP32_SPREAD)
    _check_grads(g_amp2, g_amp1, "AMP step after a full-precision step vs the first", **AMP_SPREAD)


def test_fp16_autocast_and_grad_scaler():
    c, mlp, sd, g = _ffhq_setup()
    mlp = mlp.cuda().train()
    gd = _gd()
    loss_b, g_b = _step(gd, mlp, g, torch.bfloat16)
    tr = _amp_trainer(mlp)
    loss_h, g_h = _step(gd, mlp, g, torch.float16)
    assert _amp_trainer(mlp) is tr and len(mlp._train_cache) == 1     # either autocast dtype: the same bf16 trainer
    assert abs(float(loss_h) - float(loss_b)) <= 1e-3 * abs(float(loss_b))
    _check_grads(g_h, g_b, "fp16 vs bf16 autocast", **AMP_SPREAD)
    scaler = torch.amp.GradScaler("cuda")
    opt = torch.optim.Adam(mlp.parameters(), lr=1e-4)
    with torch.autocast("cuda", dtype=torch.float16):
        loss = _latent_loss(gd, mlp, g["z0"].cuda(), g["t"].cuda(), g["noise"].cuda())
    scaler.scale(loss).backward()
    scale = float(scaler.get_scale())
    assert _amp_trainer(mlp) is tr and scale > 1
    unscaled = {k: p.grad / scale for k, p in mlp.named_parameters()}
    _check_grads(unscaled, g_b, f"GradScaler (scale {scale:g}) grads / scale vs unscaled", **AMP_SPREAD)
    before = [p.detach().clone() for p in mlp.parameters()]
    scaler.step(opt)
    scaler.update()
    assert any(not torch.equal(p, q) for p, q in zip(mlp.parameters(), before)), "GradScaler skipped a finite step"


def test_latent_diffusion_train_one_batch_under_autocast():
    from pdae_b200.utils.synth import synth_images, synth_normal
    c, mlp, sd, g = _ffhq_setup(dropout=0.1)
    mlp = mlp.cuda().train()
    enc, _ = cases.model_case({"kind": "encoder", "size": 64})
    enc = enc.cuda().requires_grad_(False).eval()
    enc.precision = "fp32"
    mean, std = (synth_normal((1, 512), 34) * 0.1).cuda(), (synth_normal((1, 512), 35).abs() + 0.5).cuda()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = _gd().latent_diffusion_train_one_batch(mlp, enc, synth_images(16, 3, 64, 33).cuda(), mean, std)["prediction_loss"]
    out.backward()
    assert torch.isfinite(out)
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in mlp.parameters())
    assert _amp_trainer(mlp).B == 16
