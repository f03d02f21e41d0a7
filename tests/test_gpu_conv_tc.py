"""wgmma/TMA convolution vs the fp32 CUDA-core kernel on identical (bf16-rounded) operands, plus the
CUDA-core kernel vs torch's CPU conv2d (the oracle's arithmetic).  Differences between the two GPU kernels can
only come from accumulation order, so the tolerance is tight."""
import pytest
import torch
import torch.nn.functional as F

from tests.util import assert_close

pytestmark = pytest.mark.gpu


def _run_conv(x, w, bias, resid, precision, k, out_dtype=torch.float32, want_stats=False, bn=0):
    from pdae_b200.engine import Plan
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    P = Plan(x.device, precision)
    out = P.new((B, H, W, Cout), out_dtype)
    out.keep = True
    st = P.conv(P.fixed(x), w, bias, out, B=B, H=H, W=W, Cin=Cin, Cout=Cout, k=k,
                residual=P.fixed(resid) if resid is not None else None, want_stats=want_stats, bn_override=bn)
    P.finalize()
    P.run()
    P.run()   # a second replay must give the same answer (persistent-kernel barriers / stats zeroing re-arm correctly)
    torch.cuda.synchronize()
    kinds = [op[0] for op in P.ops if op[0] != "zero"]
    if want_stats:  # `st` is a view into the plan's (zeroed-once-per-replay) statistics arena
        n = x.shape[0] * w.shape[0] * 2
        return out.tensor.clone(), kinds, (st.buf.tensor[st.off: st.off + n].reshape(x.shape[0], w.shape[0], 2).clone()
                                           if st is not None else None)
    return out.tensor.clone(), kinds


SHAPES = [
    # B, H, W, Cin, Cout, k, bias, residual
    (2, 16, 16, 64, 64, 3, True, False),
    (2, 16, 16, 64, 128, 3, True, True),
    (1, 32, 32, 128, 128, 3, True, True),
    (2, 8, 8, 128, 256, 3, True, False),     # tile spans 2 images
    (8, 4, 4, 256, 256, 3, True, True),      # tile spans 8 images
    (3, 8, 8, 64, 64, 3, True, True),        # batch not a multiple of the images-per-tile -> masked rows
    (2, 64, 64, 64, 64, 3, False, False),
    (1, 128, 128, 64, 128, 3, True, False),  # one tile = one image row
    (2, 16, 16, 192, 64, 1, True, True),     # 1x1 (skip / qkv / proj)
    (2, 16, 16, 64, 192, 1, True, False),
    (1, 16, 16, 1024, 512, 3, True, True),   # long K loop (144 k-blocks): pipeline wrap-around
    (2, 32, 16, 128, 64, 3, True, False),    # non-square
]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s[:6])))
def test_tc_conv_matches_simt(shape):
    B, H, W, Cin, Cout, k, has_bias, has_res = shape
    g = torch.Generator(device="cpu").manual_seed(hash(shape) % (2 ** 31))
    x = torch.randn(B, H, W, Cin, generator=g).cuda().to(torch.bfloat16)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).to(torch.bfloat16).float().cuda()
    bias = torch.randn(Cout, generator=g).cuda() if has_bias else None
    resid = torch.randn(B, H, W, Cout, generator=g).cuda() if has_res else None
    y_tc, kinds = _run_conv(x, w, bias, resid, "bf16", k)
    assert kinds == ["conv_tc2"], kinds
    y_ref, kinds = _run_conv(x, w, bias, resid, "fp32", k)
    assert kinds == ["conv2d_simt"], kinds
    assert_close(y_tc, y_ref, rtol=2e-3, atol=2e-3, what=f"tc v2 vs simt {shape}")
    # every legal N tile of the persistent kernel
    for bn in (64, 128, 256):
        if Cout % bn == 0:
            y_bn, _ = _run_conv(x, w, bias, resid, "bf16", k, bn=bn)
            assert_close(y_bn, y_ref, rtol=2e-3, atol=2e-3, what=f"tc v2 BN={bn} {shape}")
    # bf16 output + fused per-channel statistics (no residual allowed with a bf16 output)
    y_b, _, st = _run_conv(x, w, bias, None, "bf16", k, out_dtype=torch.bfloat16, want_stats=True)
    y_nores = y_ref - resid if has_res else y_ref
    assert_close(y_b.float(), y_nores, rtol=1e-2, atol=1e-2, what=f"bf16 out {shape}")
    yb = y_b.float().reshape(B, H * W, Cout)
    ref_st = torch.stack([yb.sum(1), (yb * yb).sum(1)], dim=-1)
    assert_close(st, ref_st, rtol=2e-3, atol=2e-2, what=f"fused stats {shape}")
    # fp32 output + residual + stats
    y_f, _, st = _run_conv(x, w, bias, resid, "bf16", k, want_stats=True)
    yf = y_f.reshape(B, H * W, Cout)
    assert_close(st, torch.stack([yf.sum(1), (yf * yf).sum(1)], dim=-1), rtol=2e-3, atol=2e-2, what=f"fused stats fp32 {shape}")
    # and both against torch (CPU fp32, the oracle's arithmetic)
    y_cpu = F.conv2d(x.float().cpu().permute(0, 3, 1, 2), w.cpu(), bias.cpu() if has_bias else None, padding=k // 2)
    y_cpu = y_cpu.permute(0, 2, 3, 1)
    if has_res:
        y_cpu = y_cpu + resid.cpu()
    assert_close(y_ref, y_cpu, rtol=1e-4, atol=1e-4, what=f"simt vs torch-cpu {shape}")


@pytest.mark.parametrize("cfg", [(2, 3, 16, 16, 32, 3, 1, True), (2, 64, 16, 16, 128, 3, 2, False), (1, 128, 8, 8, 3, 3, 1, False),
                                 (4, 96, 1, 1, 200, 1, 1, False)])
def test_simt_conv_general(cfg):
    """stem (NCHW in, Cin=3), stride-2 encoder conv, tiny-N, Linear (H=W=1) with SiLU on the input."""
    from pdae_b200.engine import Plan
    B, Cin, H, W, Cout, k, stride, nchw = cfg
    g = torch.Generator(device="cpu").manual_seed(7)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, generator=g)
    a_silu = (H == 1)
    ref = F.conv2d(F.silu(x) if a_silu else x, w, b, stride=stride, padding=k // 2)
    P = Plan(torch.device("cuda"), "fp32")
    xin = x.cuda().contiguous() if nchw else x.permute(0, 2, 3, 1).contiguous().cuda()
    Ho, Wo = ref.shape[2], ref.shape[3]
    out = P.new((B, Ho, Wo, Cout), torch.float32)
    out.keep = True
    P.conv(P.fixed(xin), w.cuda(), b.cuda(), out, B=B, H=H, W=W, Cin=Cin, Cout=Cout, k=k, stride=stride, in_nchw=nchw,
           a_silu=a_silu)
    P.finalize()
    P.run()
    assert_close(out.tensor.permute(0, 3, 1, 2), ref, rtol=1e-4, atol=1e-4, what=str(cfg))


@pytest.mark.parametrize("shape", [(2, 16, 16, 128, 3), (5, 8, 8, 64, 3), (1, 64, 64, 64, 6), (2, 128, 128, 128, 3)])
def test_head_conv_tensor_core(shape):
    """Image head on the tensor cores (Cout zero-padded to 16, NCHW fp32 out) vs torch."""
    from pdae_b200.engine import Plan
    B, H, W, Cin, Cout = shape
    g = torch.Generator(device="cpu").manual_seed(11)
    x = torch.randn(B, H, W, Cin, generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (3 * Cin ** 0.5)).to(torch.bfloat16).float()
    b = torch.randn(Cout, generator=g)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w, b, padding=1)
    P = Plan(torch.device("cuda"), "bf16")
    out = P.new((B, Cout, H, W), torch.float32)
    out.keep = True
    P.head_conv(P.fixed(x.cuda()), w.cuda(), b.cuda(), out, B=B, H=H, W=W, Cin=Cin, Cout=Cout)
    P.finalize()
    P.run()
    assert [o[0] for o in P.ops] == ["conv_tc2"]
    assert_close(out.tensor, ref, rtol=2e-3, atol=2e-3, what=f"tc head {shape}")


@pytest.mark.parametrize("shape", [(2, 16, 16, 128, 64, 192), (3, 8, 8, 256, 256, 512), (1, 64, 64, 64, 64, 128),
                                   (3, 24, 24, 64, 64, 64), (5, 12, 12, 64, 128, 64)])   # several images per tile AND several tiles per image
def test_fused_skip_conv(shape):
    """conv3x3(act) + conv1x1(x) + biases in ONE tensor-core launch (skip conv folded in as extra K blocks) vs torch."""
    from pdae_b200.engine import Plan
    B, H, W, Cin, Cout, Cin2 = shape
    g = torch.Generator(device="cpu").manual_seed(13)
    x = torch.randn(B, H, W, Cin, generator=g).to(torch.bfloat16)
    x2 = torch.randn(B, H, W, Cin2, generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (3 * Cin ** 0.5)).to(torch.bfloat16).float()
    w2 = (torch.randn(Cout, Cin2, 1, 1, generator=g) / Cin2 ** 0.5).to(torch.bfloat16).float()
    b, b2 = torch.randn(Cout, generator=g), torch.randn(Cout, generator=g)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w, b, padding=1) + F.conv2d(x2.float().permute(0, 3, 1, 2), w2, b2)
    ref = ref.permute(0, 2, 3, 1)
    for odt in (torch.float32, torch.bfloat16):
        P = Plan(torch.device("cuda"), "bf16")
        out = P.new((B, H, W, Cout), odt)
        out.keep = True
        st = P.conv(P.fixed(x.cuda()), w.cuda(), b.cuda(), out, B=B, H=H, W=W, Cin=Cin, Cout=Cout, k=3, want_stats=True,
                    skip=(P.fixed(x2.cuda()), w2.cuda(), b2.cuda(), Cin2))
        P.finalize()
        P.run()
        P.run()
        assert [o[0] for o in P.ops if o[0] != "zero"] == ["conv_tc2_skip"]
        tol = 2e-3 if odt == torch.float32 else 2e-2
        assert_close(out.tensor.float(), ref, rtol=tol, atol=tol, what=f"fused skip {shape} {odt}")
        y = out.tensor.float().reshape(B, H * W, Cout)
        got = st.buf.tensor[st.off: st.off + B * Cout * 2].reshape(B, Cout, 2)
        assert_close(got, torch.stack([y.sum(1), (y * y).sum(1)], dim=-1), rtol=2e-3, atol=5e-2, what="fused skip stats")


def test_head_conv_smalln():
    from pdae_b200.engine import Plan
    g = torch.Generator(device="cpu").manual_seed(9)
    for dt in (torch.float32, torch.bfloat16):
        x = torch.randn(2, 16, 16, 128, generator=g).to(dt)
        w = torch.randn(3, 128, 3, 3, generator=g) / 34.0
        b = torch.randn(3, generator=g)
        ref = F.conv2d(x.float().permute(0, 3, 1, 2), w, b, padding=1)
        P = Plan(torch.device("cuda"), "fp32")
        out = P.new((2, 3, 16, 16), torch.float32)
        out.keep = True
        P.head_conv(P.fixed(x.cuda()), w.cuda(), b.cuda(), out, B=2, H=16, W=16, Cin=128, Cout=3)
        P.finalize()
        P.run()
        assert [o[0] for o in P.ops] == ["conv3x3_smalln"]
        assert_close(out.tensor, ref, rtol=1e-4, atol=1e-4, what=f"smalln {dt}")


@pytest.mark.parametrize("T,K,batch", [(256, 128, 3), (128, 64, 5), (256, 512, 2)])
def test_softmax_gemm_epilogue(T, K, batch):
    """P = softmax_rows(alpha * Q K^T) with the softmax inside the wgmma GEMM epilogue (scores stay in registers) vs torch."""
    from pdae_b200.engine import Plan
    g = torch.Generator(device="cpu").manual_seed(17)
    q = torch.randn(batch, T, K, generator=g).to(torch.bfloat16)
    k = (torch.randn(batch, T, K, generator=g) * 1.5).to(torch.bfloat16)
    alpha = 1.0 / K ** 0.5
    ref = torch.softmax(alpha * torch.einsum("btc,bsc->bts", q.float(), k.float()), dim=-1)
    P = Plan(torch.device("cuda"), "bf16")
    out = P.new((batch, T, T), torch.bfloat16)
    out.keep = True
    P.gemm_tc(P.fixed(q.cuda()), K, T * K, P.fixed(k.cuda()), K, T * K, out, T, T * T, batch=batch, M=T, N=T, K=K,
              out_dtype=torch.bfloat16, softmax_alpha=alpha)
    P.finalize()
    P.run()
    got = out.tensor.float().cpu()
    assert_close(got, ref, rtol=1e-2, atol=2e-3, what=f"softmax gemm T={T} K={K}")        # bf16 storage of probabilities
    assert_close(got.sum(-1), torch.ones(batch, T), rtol=0, atol=6e-3, what="rows sum to 1")


@pytest.mark.parametrize("shape", [(2, 16, 16, 128, 64, 128), (1, 64, 64, 64, 64, 64), (3, 8, 8, 256, 256, 128)])
def test_fused_skip_conv_two_sources(shape):
    """The 1x1 skip conv over cat([xa, xb]) folded into conv3x3 with the two halves read through separate TMA maps."""
    from pdae_b200.engine import Plan
    B, H, W, Cin, Ca, Cb = shape
    Cout = Cin
    g = torch.Generator(device="cpu").manual_seed(19)
    x = torch.randn(B, H, W, Cin, generator=g).to(torch.bfloat16)
    xa = torch.randn(B, H, W, Ca, generator=g).to(torch.bfloat16)
    xb = torch.randn(B, H, W, Cb, generator=g).to(torch.bfloat16)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (3 * Cin ** 0.5)).to(torch.bfloat16).float()
    w2 = (torch.randn(Cout, Ca + Cb, 1, 1, generator=g) / (Ca + Cb) ** 0.5).to(torch.bfloat16).float()
    b, b2 = torch.randn(Cout, generator=g), torch.randn(Cout, generator=g)
    cat = torch.cat([xa, xb], dim=-1).float().permute(0, 3, 1, 2)
    ref = (F.conv2d(x.float().permute(0, 3, 1, 2), w, b, padding=1) + F.conv2d(cat, w2, b2)).permute(0, 2, 3, 1)
    P = Plan(torch.device("cuda"), "bf16")
    out = P.new((B, H, W, Cout), torch.float32)
    out.keep = True
    P.conv(P.fixed(x.cuda()), w.cuda(), b.cuda(), out, B=B, H=H, W=W, Cin=Cin, Cout=Cout, k=3,
           skip=((P.fixed(xa.cuda()), Ca, P.fixed(xb.cuda()), Cb), w2.cuda(), b2.cuda(), Ca + Cb))
    P.finalize()
    P.run()
    assert_close(out.tensor, ref, rtol=2e-3, atol=2e-3, what=f"two-source fused skip {shape}")


@pytest.mark.parametrize("shape", [(3, 3, 32, 32, 64), (2, 1, 16, 40, 32), (2, 3, 64, 64, 128)])
def test_stem_conv_bf16_with_stats(shape):
    """Image stem: NCHW fp32 -> bf16 NHWC stream + per-channel sums of the stored values, vs torch."""
    from pdae_b200.engine import Plan, _STREAM
    B, Cin, H, W, Cout = shape
    g = torch.Generator(device="cpu").manual_seed(23)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / (3 * Cin ** 0.5)
    b = torch.randn(Cout, generator=g)
    ref = F.conv2d(x, w, b, padding=1).permute(0, 2, 3, 1)
    P = Plan(torch.device("cuda"), "bf16")
    out = P.new((B, H, W, Cout), torch.bfloat16)
    out.keep = True
    st = P.new_stats(B, Cout)
    wp = P.fixed(w.reshape(Cout, Cin, 9).permute(2, 1, 0).contiguous().cuda())
    P.call("stem_conv_bf16", P.fixed(x.cuda()), wp, P.fixed(b.cuda()), out, st, B, H, W, Cin, Cout, _STREAM)
    P.finalize()
    P.run()
    P.run()     # the statistics arena is re-zeroed on every replay
    assert_close(out.tensor.float(), ref, rtol=1e-2, atol=1e-2, what=f"stem {shape}")
    y = out.tensor.float().reshape(B, H * W, Cout)
    got = st.buf.tensor[st.off: st.off + B * Cout * 2].reshape(B, Cout, 2)
    assert_close(got, torch.stack([y.sum(1), (y * y).sum(1)], dim=-1), rtol=2e-3, atol=5e-2, what="stem stats")
