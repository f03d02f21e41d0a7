"""Attention under torch.autocast in training: the transposed-operand batched GEMMs and the softmax-gradient GEMM through the
C-ABI against float64 references, a lone AttentionBlock's bf16 training step and whole PDAE / 128-px encoder steps against
oracle autograd on the CPU, and the plans actually recorded (eligible blocks on the tensor cores, T = 64 blocks and 32-channel
heads on the CUDA-core path, full-precision plans unchanged)."""
import copy
import ctypes
import math

import pytest
import torch

from oracle import pdae_oracle as O
from pdae_b200 import _native
from tests import cases
from tests.test_gpu_encoder_amp import ENC_KIND, _enc_inputs, _enc_step, _encoder
from tests.test_gpu_encoder_amp import _to_train as _enc_to_train
from tests.test_gpu_training_amp import (AMP_SPREAD, FP32_SPREAD, SHIFT_CFG, T_STEPS, _check_grads, _gd, _shift_inputs,
                                         _shift_module, _shift_step)
from tests.test_gpu_training_amp import _to_train as _dec_to_train

pytestmark = pytest.mark.gpu
DEV = "cuda"
SIMT_ATTN_FWD = ("attention_simt",)
SIMT_ATTN_BWD = ("gemm_batched_simt", "softmax_bwd")


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _elem(t, off):
    """Pointer to element `off` of a contiguous tensor."""
    return ctypes.c_void_p(t.data_ptr() + off * t.element_size())


def _run(create, *args):
    L = _native.lib()
    h = ctypes.c_void_p()
    _native.check(getattr(L, create)(ctypes.byref(h), *args), create)
    try:
        _native.check(L.pdae_conv_tc2_run(h, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "pdae_conv_tc2_run")
        torch.cuda.synchronize()
    finally:
        L.pdae_conv_tc2_destroy(h)


def _offsets(legacy, C, ch):
    """(head stride, K offset, V offset) inside a qkv row, as AttentionBlock.emit / Backward.attention use them."""
    return (3 * ch, ch, 2 * ch) if legacy else (ch, C, 2 * C)


# ---- 1. transposed-operand GEMMs ------------------------------------------------------------------------------------------
GEMM_CASES = [(T, ch, legacy) for T in (128, 256) for ch in (64, 256, 384, 512) for legacy in (True, False)]


@pytest.mark.parametrize("T,ch,legacy", GEMM_CASES)
def test_transposed_gemms_match_float64_matmul(T, ch, legacy):
    """dV = P^T dO (A, B MN-major), dQ = dS K (B MN-major), dK = dS^T Q (A, B MN-major) on the strided qkv layout of two heads,
    written into one fp32 d_qkv; against float64 matmul of the same bf16 values."""
    B, heads = 2, 2
    C = heads * ch
    hs, ko, vo = _offsets(legacy, C, ch)
    g = torch.Generator(device="cpu").manual_seed(T + ch + legacy)
    qkv = torch.randn(B, T, 3 * C, generator=g).to(torch.bfloat16).to(DEV)
    d_o = (torch.randn(B, T, C, generator=g) * 0.1).to(torch.bfloat16).to(DEV)
    probs = torch.softmax(torch.randn(B * heads, T, T, generator=g) * 2, -1).to(torch.bfloat16).to(DEV)
    d_s = (torch.randn(B * heads, T, T, generator=g) * 0.01).to(torch.bfloat16).to(DEV)
    d_qkv = torch.full((B, T, 3 * C), float("nan"), device=DEV)
    row, TT = 3 * C, T * T
    for h in range(heads):
        q, k, v, o = h * hs, h * hs + ko, h * hs + vo, h * ch
        _run("pdae_gemm_tc2_create_major", _elem(probs, h * TT), 1, T, heads * TT, _elem(d_o, o), 1, C, T * C,
             _elem(d_qkv, v), row, T * row, B, T, ch, T)
        _run("pdae_gemm_tc2_create_major", _elem(d_s, h * TT), 0, T, heads * TT, _elem(qkv, k), 1, row, T * row,
             _elem(d_qkv, q), row, T * row, B, T, ch, T)
        _run("pdae_gemm_tc2_create_major", _elem(d_s, h * TT), 1, T, heads * TT, _elem(qkv, q), 1, row, T * row,
             _elem(d_qkv, k), row, T * row, B, T, ch, T)
    assert torch.isfinite(d_qkv).all(), "an element of d_qkv was not written"
    q64, d64, p64, s64 = qkv.double(), d_o.double(), probs.double().view(B, heads, T, T), d_s.double().view(B, heads, T, T)
    for h in range(heads):
        q, k, v, o = h * hs, h * hs + ko, h * hs + vo, h * ch
        refs = {"dV": (v, p64[:, h].transpose(1, 2) @ d64[..., o:o + ch]),
                "dQ": (q, s64[:, h] @ q64[..., k:k + ch]),
                "dK": (k, s64[:, h].transpose(1, 2) @ q64[..., q:q + ch])}
        for what, (off, ref) in refs.items():
            got = d_qkv[..., off:off + ch].double()
            err, scale = (got - ref).abs().max().item(), ref.abs().max().item()
            print(f"T={T} ch={ch} {'legacy' if legacy else 'new'} head {h} {what}: max|err| {err / scale:.2e} of max|ref|")
            assert err <= 2e-5 * scale, (what, h, err, scale)


def test_gemm_with_mn_major_a_and_k_major_b():
    """The remaining combination (A MN-major, B K-major), and N = 2 n-tiles."""
    B, M, N, K = 3, 256, 256, 128
    g = torch.Generator(device="cpu").manual_seed(11)
    a = torch.randn(B, K, M, generator=g).to(torch.bfloat16).to(DEV)        # A_i stored [K][M]
    b = torch.randn(B, N, K, generator=g).to(torch.bfloat16).to(DEV)        # B_i stored [N][K]
    out = torch.full((B, M, N), float("nan"), device=DEV)
    _run("pdae_gemm_tc2_create_major", _p(a), 1, M, K * M, _p(b), 0, K, N * K, _p(out), N, M * N, B, M, N, K)
    ref = a.double().transpose(1, 2) @ b.double().transpose(1, 2)
    err, scale = (out.double() - ref).abs().max().item(), ref.abs().max().item()
    assert err <= 2e-5 * scale, (err, scale)


# ---- 2. softmax-gradient GEMM ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [64, 128, 256])
@pytest.mark.parametrize("ch", [64, 128])
def test_softmax_grad_gemm_matches_float64(N, ch):
    """dS = alpha P (dP - rowsum(P dP)), dP = dO V^T, on a strided (legacy-order) qkv layout of two heads: within one bf16 ulp of
    each element plus 2e-5 of the largest, against float64 from the same bf16 P, dO and V."""
    B, heads, M = 2, 2, 256
    C = heads * ch
    hs, ko, vo = _offsets(True, C, ch)
    alpha = 1.0 / math.sqrt(ch)
    g = torch.Generator(device="cpu").manual_seed(N + ch)
    qkv = torch.randn(B, N, 3 * C, generator=g).to(torch.bfloat16).to(DEV)   # V rows = the N keys
    d_o = (torch.randn(B, M, C, generator=g) * 0.1).to(torch.bfloat16).to(DEV)
    probs = torch.softmax(torch.randn(B * heads, M, N, generator=g) * 2, -1).to(torch.bfloat16).to(DEV)
    d_s = torch.full((B * heads, M, N), float("nan"), device=DEV).to(torch.bfloat16)
    MN = M * N
    for h in range(heads):
        _run("pdae_gemm_tc2_softmax_grad_create", _elem(d_o, h * ch), C, M * C, _elem(qkv, h * hs + vo), 3 * C, N * 3 * C,
             _elem(probs, h * MN), N, heads * MN, _elem(d_s, h * MN), N, heads * MN, B, M, N, ch, ctypes.c_float(alpha))
    p64 = probs.double().view(B, heads, M, N)
    got = d_s.double().view(B, heads, M, N)
    assert torch.isfinite(got).all()
    for h in range(heads):
        dp = d_o.double()[..., h * ch:(h + 1) * ch] @ qkv.double()[..., h * hs + vo:h * hs + vo + ch].transpose(1, 2)
        ph = p64[:, h]
        ref = alpha * ph * (dp - (ph * dp).sum(-1, keepdim=True))
        ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(1e-30))) - 7)
        err = (got[:, h] - ref).abs()
        excess = (err - ulp - 2e-5 * ref.abs().max()).max().item()
        print(f"N={N} ch={ch} head {h}: max|err| {err.max().item():.3e}, max|ref| {ref.abs().max().item():.3e}")
        assert excess <= 0, excess


# ---- 3. a lone AttentionBlock ---------------------------------------------------------------------------------------------
def _block_step(blk, x, dy, amp=True):
    """Training forward + backward of one AttentionBlock through the trainers' plan machinery: returns (y, {param name: grad},
    dx, forward ops, backward ops)."""
    from pdae_b200.engine import Plan
    from pdae_b200.model.module import Src
    from pdae_b200.train import Backward, GradSink, bwd_plan
    dev = torch.device(DEV)
    B, C, H, W = x.shape
    P = Plan(dev, "fp32")
    P.keep_all = True
    P.train_tc = "bf16" if amp else "bf16x3"
    xin = P.new((B, H, W, C), torch.float32, "x")
    xin.keep = True
    tape = []
    y = blk.emit(P, Src(xin, C, B, H, W), tape=tape)
    y.b1.keep = True
    P.finalize()
    BP = bwd_plan(dev, amp)
    sink = GradSink()
    bw = Backward(BP, sink)
    d_in = BP.new((B, H, W, C), torch.float32, "dy")
    d_in.keep = True
    (kind, mod, sv), = tape
    dx = bw.attention(mod, sv, d_in)
    dx.keep = True
    BP.finalize()
    xin.tensor.copy_(x.permute(0, 2, 3, 1))
    P.run()
    d_in.tensor.copy_(dy.permute(0, 2, 3, 1))
    BP.run()
    grads = sink.collect()
    torch.cuda.synchronize()
    named = {k: grads[id(p)].clone() for k, p in blk.named_parameters()}
    return (y.b1.tensor.permute(0, 3, 1, 2).float().cpu(), named, dx.tensor.permute(0, 3, 1, 2).cpu(),
            [fn for fn, _ in P.ops], [fn for fn, _ in BP.ops])


@pytest.mark.parametrize("heads", [1, 4])
@pytest.mark.parametrize("new_order", [False, True])
def test_attention_block_step_under_bf16_matches_oracle(heads, new_order):
    from pdae_b200.model.module import AttentionBlock
    from pdae_b200.utils.synth import fill_module_
    B, C, H = 2, 256, 16
    blk = fill_module_(AttentionBlock(C, heads, -1, new_order), seed=9 + heads)
    x = torch.randn(B, C, H, H, generator=torch.Generator().manual_seed(4)) * 1.5
    dy = torch.randn(B, C, H, H, generator=torch.Generator().manual_seed(5)) * 0.1
    sd = {k: v.requires_grad_(True) for k, v in cases.sd_of(blk).items()}
    xr = x.clone().requires_grad_(True)
    sdp = {"a." + k: v for k, v in sd.items()}
    y_ref = O.attention_block(sdp, "a", xr, heads, new_order)
    y_ref.backward(dy)
    blk = blk.cuda().train()
    y, grads, dx, fwd_ops, bwd_ops = _block_step(blk, x.to(DEV), dy.to(DEV))
    r = float((y.double() - y_ref.detach().double()).norm() / y_ref.detach().double().norm())
    print(f"AttentionBlock heads={heads} {'new' if new_order else 'legacy'} order, bf16: y rel-L2 {r:.2e}")
    assert r <= 5e-2
    _check_grads(dict(grads, dx=dx), dict({k: v.grad for k, v in sd.items()}, dx=xr.grad),
                 f"AttentionBlock heads={heads} {'new' if new_order else 'legacy'} bf16 vs oracle")
    assert not any(fn in SIMT_ATTN_FWD for fn in fwd_ops)
    assert not any(fn in SIMT_ATTN_BWD for fn in bwd_ops)
    assert fwd_ops.count("gemm_tc2_softmax") == heads
    assert bwd_ops.count("gemm_tc2_softmax_grad") == heads and bwd_ops.count("gemm_tc2_major") == 3 * heads


# ---- 4. + 5. whole steps and the recorded plans ----------------------------------------------------------------------------
def _attn_ops(plan):
    ops = [fn for fn, _ in plan.ops]
    return {fn: ops.count(fn) for fn in SIMT_ATTN_FWD + SIMT_ATTN_BWD + ("gemm_tc2_softmax", "gemm_tc2_softmax_grad",
                                                                          "gemm_tc2_major")}


def test_pdae_step_under_bf16_autocast_runs_the_tensor_core_attention():
    """The existing AMP test config: attention at 16x16 (T = 256, one head of 128) in the two shift output blocks, and at 8x8
    (T = 64, the middle block) which stays on the CUDA-core path."""
    dec0 = _shift_module()
    inputs = _shift_inputs()
    x0, noise, z = inputs
    dsd = {k: v.requires_grad_(k.startswith(("label_emb", "shift_"))) for k, v in cases.sd_of(dec0).items()}
    zr = z.clone().requires_grad_(True)
    ref_loss = O.DiffusionOracle(cases.DIFF).representation_learning_loss(
        lambda x: zr, lambda x, t, zz: O.shiftunet_forward(dsd, SHIFT_CFG, x, t, zz), x0, T_STEPS, noise)
    ref_loss.backward()
    dec = _dec_to_train(dec0)
    loss, grads, gz = _shift_step(_gd(), dec, inputs, torch.bfloat16)
    r = abs(float(loss) - float(ref_loss)) / abs(float(ref_loss))
    print(f"bf16 autocast PDAE step: loss rel {r:.2e}")
    assert r <= 1e-2
    _check_grads(dict(grads, z=gz), dict({k: v.grad for k, v in dsd.items() if v.grad is not None}, z=zr.grad),
                 "ShiftUNet with tensor-core attention, bf16 autocast vs oracle")
    tr = [t for t in dec._train_cache.values() if t.amp][0]
    f, b = _attn_ops(tr.fwd), _attn_ops(tr.bwd)
    print("forward attention ops", f, "backward", b)
    assert f["attention_simt"] == 1                              # the 8x8 middle block only
    assert b["gemm_batched_simt"] == 4 and b["softmax_bwd"] == 1
    assert f["gemm_tc2_softmax"] == 2                            # two eligible 16x16 blocks, one head each
    assert b["gemm_tc2_softmax_grad"] == 2 and b["gemm_tc2_major"] == 6


def test_encoder_128_step_under_bf16_autocast_runs_the_tensor_core_attention():
    size = 128
    enc0 = _encoder(size)
    inputs = _enc_inputs(size)
    esd = {k: v.requires_grad_(True) for k, v in cases.sd_of(enc0).items()}
    z_ref = O.encoder_forward(esd, ENC_KIND[size], inputs[0])
    (z_ref * inputs[1]).sum().backward()
    enc = _enc_to_train(enc0)
    z, grads = _enc_step(enc, inputs, torch.bfloat16)
    r = float((z.double().cpu() - z_ref.detach().double()).norm() / z_ref.detach().double().norm())
    print(f"128-px encoder under bf16 autocast: z rel-L2 {r:.2e}")
    assert r <= 5e-2
    _check_grads(grads, {k: v.grad for k, v in esd.items()}, "128-px encoder with tensor-core attention vs oracle")
    tr = [t for t in enc._train_cache.values() if t.amp][0]
    f, b = _attn_ops(tr.fwd), _attn_ops(tr.bwd)
    print("forward attention ops", f, "backward", b)
    assert f["attention_simt"] == 0 and b["gemm_batched_simt"] == 0 and b["softmax_bwd"] == 0
    assert f["gemm_tc2_softmax"] > 0 and b["gemm_tc2_softmax_grad"] == f["gemm_tc2_softmax"]


def test_celeba64_encoder_keeps_the_cuda_core_attention():
    """32-channel heads are not eligible: the AMP plans of the 64-px encoder record the CUDA-core attention as before."""
    enc = _enc_to_train(_encoder(64))
    _enc_step(enc, _enc_inputs(64), torch.bfloat16)
    tr = [t for t in enc._train_cache.values() if t.amp][0]
    f, b = _attn_ops(tr.fwd), _attn_ops(tr.bwd)
    assert f["attention_simt"] > 0 and b["softmax_bwd"] == f["attention_simt"]
    assert f["gemm_tc2_softmax"] == 0 and b["gemm_tc2_softmax_grad"] == 0 and b["gemm_tc2_major"] == 0


def _op_sig(plan):
    return [(fn, [(x.shape, x.dtype) if hasattr(x, "shape") else None for x in args]) for fn, args in plan.ops]


def test_full_precision_plans_and_grad_scaler_with_tensor_core_attention():
    """The 128-px encoder (eligible attention): its full-precision trainer after AMP steps records exactly the plans of an
    encoder that never saw autocast, and GradScaler as the reference trainer uses it yields finite, unscaled-equivalent grads."""
    enc = _enc_to_train(_encoder(128))
    fresh = copy.deepcopy(enc)
    inputs = _enc_inputs(128)
    _, g_ref = _enc_step(fresh, inputs)
    _, g_amp = _enc_step(enc, inputs, torch.bfloat16)
    _, g_full = _enc_step(enc, inputs)
    full_tr = [t for t in enc._train_cache.values() if not t.amp][0]
    fresh_tr = list(fresh._train_cache.values())[0]
    for a, b in ((full_tr.fwd, fresh_tr.fwd), (full_tr.bwd, fresh_tr.bwd)):
        assert a.precision == b.precision and a.train_tc == b.train_tc
        assert _op_sig(a) == _op_sig(b)
    assert _attn_ops(full_tr.fwd)["gemm_tc2_softmax"] == 0 and _attn_ops(full_tr.bwd)["gemm_tc2_softmax_grad"] == 0
    _check_grads(g_full, g_ref, "full precision after AMP vs never-autocast encoder", **FP32_SPREAD)
    scaler = torch.amp.GradScaler("cuda")
    opt = torch.optim.Adam(list(enc.parameters()), lr=1e-4)
    _, g_s = _enc_step(enc, inputs, torch.float16, scaler=scaler)
    scale = float(scaler.get_scale())
    assert scale > 1 and all(torch.isfinite(g).all() for g in g_s.values())
    _check_grads({k: g / scale for k, g in g_s.items()}, g_amp, f"GradScaler (scale {scale:g}) grads / scale vs unscaled",
                 **AMP_SPREAD)
    before = [p.detach().clone() for p in enc.parameters()]
    scaler.step(opt)
    scaler.update()
    assert any(not torch.equal(p, q) for p, q in zip(enc.parameters(), before)), "GradScaler skipped a finite step"
