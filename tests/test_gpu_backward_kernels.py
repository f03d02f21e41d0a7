"""Backward CUDA-core kernels through the C-ABI vs float64 on the device: conv data gradient (generic tile kernel, the
3-channel image-head kernel, the split-K wide-Linear kernel), the bias-gradient column sum (vector and scalar paths), the
split-K conv weight gradient (NHWC / NCHW input, SiLU on the input, the Linear-bank shape, accumulation into dw), the batched
attention GEMM (all transposes, both qkv channel orders), softmax backward, embedding backward with repeated classes, and the
dsilu_mul / add_inplace / nchw_to_nhwc helpers."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from pdae_b200 import _native

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,stride", [
    (3, 16, 16, 64, 3, 3, 1),        # image head: 3x3 onto 3 channels (conv3x3_dgrad_smalln)
    (2, 9, 7, 32, 4, 3, 1),          # same kernel, odd image, 4 output channels
    (5, 1, 1, 96, 2048, 1, 1),       # wide Linear: split-K kernel, ragged batch block
    (33, 1, 1, 512, 1100, 1, 1),     # wide Linear: two batch blocks, ragged last weight chunk
    (2, 8, 8, 32, 48, 3, 2),         # generic tile kernel (stride 2)
])
def test_conv_dgrad_matches_float64_autograd(B, H, W, Cin, Cout, k, stride):
    g = torch.Generator().manual_seed(5)
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (k * Cin ** 0.5)).to(DEV)
    dy = torch.randn(B, Ho, Wo, Cout, generator=g).to(DEV)
    wt = w.reshape(Cout, Cin, k * k).permute(2, 0, 1).contiguous()             # [k*k][Cout][Cin]
    dx = torch.full((B, H, W, Cin), float("nan"), device=DEV)
    L = _native.lib()
    _native.check(L.pdae_conv2d_dgrad_simt(_p(dy), _p(wt), _p(dx), B, H, W, Cin, Cout, k, stride, pad, 0, _stream()), "dgrad")
    torch.cuda.synchronize()
    x = torch.zeros(B, Cin, H, W, device=DEV, dtype=torch.float64, requires_grad=True)
    F.conv2d(x, w.double(), stride=stride, padding=pad).backward(dy.double().permute(0, 3, 1, 2))
    ref = x.grad.permute(0, 2, 3, 1)
    err = (dx.double() - ref).abs().max().item()
    assert err <= 2e-5 * ref.abs().max().item() + 1e-6, err


@pytest.mark.parametrize("M,N", [(4096, 128), (1000, 64), (37, 512), (70000, 256), (513, 3), (32, 2052)])
def test_colsum_matches_float64(M, N):
    g = torch.Generator().manual_seed(9)
    dy = torch.randn(M, N, generator=g).to(DEV)
    out = torch.zeros(N, device=DEV)
    _native.check(_native.lib().pdae_colsum(_p(dy), ctypes.c_int64(M), N, _p(out), _stream()), "colsum")
    torch.cuda.synchronize()
    ref = dy.double().sum(0)
    assert (out.double() - ref).abs().max().item() <= 1e-5 * (M ** 0.5) * 4 + 1e-6


def _cdiv(a, b):
    return (a + b - 1) // b


# conv_wgrad_kernel's tile (DBM rows of dw x DBN output channels, DBK pixels per k-step, backward_simt.cu) and the CTA count
# its host code aims for (148 SMs x 4)
WG_DBM, WG_DBN, WG_DBK, WG_TARGET_CTAS = 64, 64, 16, 148 * 4


def _wgrad_chunk(P, MK, Cout):
    """Split-K pixel chunk and slice count of pdae_conv2d_wgrad_simt (its host code): they size the tolerance, and tell
    whether the last slice is ragged."""
    cells = _cdiv(MK, WG_DBM) * _cdiv(Cout, WG_DBN)
    splits = min((WG_TARGET_CTAS + cells - 1) // cells, _cdiv(P, 256), 65535)
    splits = max(splits, 1)
    chunk = _cdiv(_cdiv(P, splits), WG_DBK) * WG_DBK
    return chunk, _cdiv(P, chunk)


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,stride,nchw,a_silu,ragged", [
    (2, 9, 7, 20, 36, 3, 1, 0, 0, False),       # 3x3, NHWC, ragged tiles in both dw dimensions
    (3, 13, 11, 32, 70, 3, 2, 1, 1, False),     # stride 2, NCHW input, SiLU applied to the input
    (2, 16, 16, 64, 64, 1, 1, 0, 1, False),     # 1x1 with SiLU
    (3, 17, 15, 3, 64, 3, 2, 1, 0, False),      # image input (3 channels, NCHW), stride 2
    (6, 1, 1, 128, 1100, 1, 1, 0, 1, False),    # the Linear bank of train.py: (B,1,1,E -> total), SiLU(emb) input
    (1, 33, 31, 16, 8, 3, 1, 0, 1, True),       # 1023 pixels in four 256-pixel slices: the last one is ragged (255)
])
def test_conv_wgrad_matches_float64_autograd(B, H, W, Cin, Cout, k, stride, nchw, a_silu, ragged):
    g = torch.Generator().manual_seed(13)
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    x = torch.randn(B, Cin, H, W, generator=g).to(DEV)
    dy = torch.randn(B, Ho, Wo, Cout, generator=g).to(DEV)
    dw0 = torch.randn(k * k * Cin, Cout, generator=g).to(DEV)        # dw accumulates: += onto what is there
    dw = dw0.clone()
    xin = x.contiguous() if nchw else x.permute(0, 2, 3, 1).contiguous()
    _native.check(_native.lib().pdae_conv2d_wgrad_simt(_p(xin), nchw, a_silu, _p(dy), _p(dw), B, H, W, Cin, Cout, k, stride, pad,
                                                       _stream()), "wgrad")
    torch.cuda.synchronize()
    a = F.silu(x.double()) if a_silu else x.double()
    dyn = dy.double().permute(0, 3, 1, 2)

    def wg(inp, grad):   # [Cout][Cin][k][k] -> dw layout [k*k*Cin][Cout]
        w = torch.nn.grad.conv2d_weight(inp, (Cout, Cin, k, k), grad, stride=stride, padding=pad)
        return w.permute(2, 3, 1, 0).reshape(k * k * Cin, Cout)
    ref = wg(a, dyn)
    mag = wg(a.abs(), dyn.abs())
    P = B * Ho * Wo
    chunk, slices = _wgrad_chunk(P, k * k * Cin, Cout)
    assert not ragged or (slices > 1 and P % chunk != 0), f"P={P}, chunk={chunk}: no longer a ragged last split-K slice"
    # per CTA an fp32 fma chain over its chunk, then one fp32 atomic per slice onto dw; SiLU(x) within 4u
    tol = (chunk + slices + 8) * 2.0 ** -24 * (mag + dw0.double().abs())
    err = (dw.double() - dw0.double() - ref).abs()
    ratio = (err / tol).max().item()
    print(f"[ratio] wgrad B={B} {H}x{W} {Cin}->{Cout} k={k} s={stride} nchw={nchw} silu={a_silu} "
          f"(P={P}, chunk={chunk}, tail={P % chunk}): {ratio:.3e}")
    assert ratio <= 1.0, ratio


@pytest.mark.parametrize("legacy", [1, 0], ids=["legacy_order", "new_order"])
@pytest.mark.parametrize("tA,tB", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_gemm_batched_matches_float64(tA, tB, legacy):
    """C[b,h] = alpha op(A[b,h]) op(B[b,h]) with B a per-head column block of a [batch][T][3C] qkv-like buffer (head stride
    3ch in the legacy channel order, ch in the new one), and C likewise when its columns are the head channels."""
    g = torch.Generator().manual_seed(17 + 2 * tA + tB)
    batch, heads, ch, T, M = 2, 3, 20, 45, 37       # none of M, N, K is a multiple of the 64 x 64 x 16 tile
    C = heads * ch
    hs, ko = (3 * ch, ch) if legacy else (ch, C)
    alpha = 0.7
    K, N = (ch, T) if tB else (T, ch)
    qkv = torch.randn(batch, T, 3 * C, generator=g).to(DEV)
    b_off, ldb, b_bs, b_hs = ko, 3 * C, T * 3 * C, hs
    ra, ca = (K, M) if tA else (M, K)
    lda = ca + 3
    Abuf = torch.randn(batch, heads, ra, lda, generator=g).to(DEV)
    a_bs, a_hs = heads * ra * lda, ra * lda
    if N == ch:       # output columns are head channels: a column block of a [batch][M][3C] buffer
        ldc, c_off, c_bs, c_hs = 3 * C, 2 * C if not legacy else 2 * ch, M * 3 * C, hs
        Cbuf = torch.full((batch, M, 3 * C), float("nan"), device=DEV)
    else:
        ldc, c_off, c_bs, c_hs = N + 5, 0, heads * M * (N + 5), M * (N + 5)
        Cbuf = torch.full((batch, heads, M, N + 5), float("nan"), device=DEV)
    _native.check(_native.lib().pdae_gemm_batched_simt(
        _p(Abuf), lda, a_bs, a_hs, tA, ctypes.c_void_p(qkv.data_ptr() + 4 * b_off), ldb, b_bs, b_hs, tB,
        ctypes.c_void_p(Cbuf.data_ptr() + 4 * c_off), ldc, c_bs, c_hs, M, N, K, batch, heads, alpha, _stream()), "gemm_batched")
    torch.cuda.synchronize()
    Af, Bf = Abuf.double().flatten(), qkv.double().flatten()
    want = torch.full_like(Cbuf, float("nan"), dtype=torch.float64).flatten()
    tol = torch.zeros_like(want)
    for b in range(batch):
        for h in range(heads):
            ao = b * a_bs + h * a_hs
            Aop = Af.as_strided((M, K), (1, lda) if tA else (lda, 1), ao)
            bo = b_off + b * b_bs + h * b_hs
            Bop = Bf.as_strided((K, N), (1, ldb) if tB else (ldb, 1), bo)
            co = c_off + b * c_bs + h * c_hs
            want.as_strided((M, N), (ldc, 1), co).copy_(alpha * Aop @ Bop)
            tol.as_strided((M, N), (ldc, 1), co).copy_((K + 1) * 2.0 ** -24 * alpha * (Aop.abs() @ Bop.abs()))
    got = Cbuf.double().flatten()
    written = ~torch.isnan(want)
    assert torch.equal(torch.isnan(got), ~written), "elements outside the output blocks were written (or some were not)"
    ratio = ((got[written] - want[written]).abs() / tol[written]).max().item()
    print(f"[ratio] gemm_batched tA={tA} tB={tB} legacy={legacy}: {ratio:.3e}")
    assert ratio <= 1.0, ratio


@pytest.mark.parametrize("cols", [4, 33, 1024])
def test_softmax_bwd_matches_float64(cols):
    g = torch.Generator().manual_seed(cols)
    rows, spare = 43, 8           # 43 rows: the last CTA's warps past row 42 return early
    P = torch.softmax(torch.randn(rows + spare, cols, generator=g), dim=1).to(DEV)
    d0 = torch.randn(rows + spare, cols, generator=g).to(DEV)
    dP = d0.clone()
    alpha = 0.125
    _native.check(_native.lib().pdae_softmax_bwd(_p(P), _p(dP), ctypes.c_int64(rows), cols, alpha, _stream()), "softmax_bwd")
    torch.cuda.synchronize()
    assert torch.equal(dP[rows:], d0[rows:]), "rows past the end were written"
    p, d = P[:rows].double(), d0[:rows].double()
    s = (p * d).sum(1, keepdim=True)
    ref = alpha * p * (d - s)
    u = 2.0 ** -24
    ds = (cols // 32 + 7) * u * (p * d).abs().sum(1, keepdim=True)   # per-lane fma chain + five shuffle adds
    tol = alpha * p * (ds + u * (d.abs() + s.abs())) + 3 * u * ref.abs() + 1e-300
    ratio = ((dP[:rows].double() - ref).abs() / tol).max().item()
    print(f"[ratio] softmax_bwd cols={cols}: {ratio:.3e}")
    assert ratio <= 1.0, ratio


def test_embedding_bwd_sums_duplicate_indices():
    g = torch.Generator().manual_seed(21)
    B, E, ncls = 37, 130, 5
    idx = torch.tensor([i % 3 for i in range(B - 2)] + [4, 4], dtype=torch.int64).to(DEV)   # class 3 never used
    d = torch.randn(B, E, generator=g).to(DEV)
    dw0 = torch.randn(ncls, E, generator=g).to(DEV)
    dw = dw0.clone()
    _native.check(_native.lib().pdae_embedding_bwd(_p(d), _p(idx), _p(dw), B, E, _stream()), "embedding_bwd")
    torch.cuda.synchronize()
    ref = dw0.double().index_add(0, idx, d.double())
    mag = dw0.double().abs().index_add(0, idx, d.double().abs())
    cnt = torch.bincount(idx, minlength=ncls).double()[:, None]
    tol = (cnt + 1) * 2.0 ** -24 * mag
    assert torch.equal(dw[3], dw0[3])
    ratio = ((dw.double() - ref).abs() / tol.clamp_min(1e-300)).max().item()
    print(f"[ratio] embedding_bwd: {ratio:.3e}")
    assert ratio <= 1.0, ratio


def test_elementwise_backward_helpers_match_float64():
    """dsilu_mul, add_inplace and nchw_to_nhwc at sizes that are not multiples of the 256-thread CTA."""
    g = torch.Generator().manual_seed(23)
    L = _native.lib()
    n = 12345
    gr = torch.randn(n, generator=g).to(DEV)
    x = (3 * torch.randn(n, generator=g)).to(DEV)
    out = torch.full((n + 3,), float("nan"), device=DEV)
    _native.check(L.pdae_dsilu_mul(_p(gr), _p(x), _p(out), ctypes.c_int64(n), _stream()), "dsilu_mul")
    a0 = torch.randn(n + 3, generator=g).to(DEV)
    b = torch.randn(n, generator=g).to(DEV)
    a = a0.clone()
    _native.check(L.pdae_add_inplace(_p(a), _p(b), ctypes.c_int64(n), _stream()), "add_inplace")
    Bn, Cn, HW = 3, 5, 63
    src = torch.randn(Bn, Cn, HW, generator=g).to(DEV)
    dst = torch.full((Bn, HW, Cn), float("nan"), device=DEV)
    _native.check(L.pdae_nchw_to_nhwc(_p(src), _p(dst), Bn, Cn, HW, _stream()), "nchw_to_nhwc")
    torch.cuda.synchronize()
    xd = x.double()
    sg = torch.sigmoid(xd)
    ref = gr.double() * sg * (1 + xd * (1 - sg))
    u = 2.0 ** -24
    # sigmoid via expf and a division (3u), then s(1 + x(1 - s)): 1 - s carries s's absolute error times |x|
    tol = 8 * u * (1 + xd.abs()) * gr.double().abs() + u * ref.abs() + 1e-300
    ratio = ((out[:n].double() - ref).abs() / tol).max().item()
    print(f"[ratio] dsilu_mul: {ratio:.3e}")
    assert ratio <= 1.0, ratio
    assert torch.isnan(out[n:]).all()
    assert torch.equal(a[:n], a0[:n] + b) and torch.equal(a[n:], a0[n:])       # fp32 add is correctly rounded: bit exact
    assert torch.equal(dst, src.permute(0, 2, 1))
