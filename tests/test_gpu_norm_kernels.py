"""GroupNorm kernels through the C-ABI vs float64 torch on the device, at the channel counts, concats and image sizes of the
production configs: statistics (gn_stats / ch_stats), coefficients (gn_coef / gn_coef_ch), the forward apply (gn_apply in
every dtype combination, both its 8-wide and generic paths; gn_apply_split3) and the three backward passes (gn_bwd_sums ->
gn_bwd_coef -> gn_bwd_apply, in the order of train.Backward.gn).

The reference is GroupNorm(32, eps=1e-5) of cat(x1, x2), then (.)*(1+e_s)+e_sh, then (.)*(1+z_s)+z_sh, then SiLU, then
nearest-up x2 or avg_pool2d(2).  Every tolerance is a worst-case bound of the kernel's fp32 arithmetic (u = 2^-24 per
rounding, a recursive fp32 sum of n terms is off by at most n*u*sum|terms|), evaluated per element in float64 from the
magnitudes of the terms; the comments next to each bound say where it comes from.  Outputs are filled with NaN (fp32) or
0xFFFF (bf16, also a NaN) before each launch, so that an element the kernel never writes fails the comparison."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from pdae_b200 import _native
from pdae_b200._native import PDAE_BF16, PDAE_F32, RESAMPLE_DOWN2, RESAMPLE_NONE, RESAMPLE_UP2

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24          # fp32 unit roundoff
EPS = 1e-5
RS_NAMES = {RESAMPLE_NONE: "none", RESAMPLE_UP2: "up2", RESAMPLE_DOWN2: "down2"}
DT = {PDAE_F32: torch.float32, PDAE_BF16: torch.bfloat16}


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _L():
    return _native.lib()


def _nan(shape, dtype=torch.float32):
    if dtype == torch.bfloat16:
        return torch.full(shape, -1, dtype=torch.int16, device=DEV).view(torch.bfloat16)   # 0xFFFF: a bf16 NaN
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def _report(name, err, tol):
    """Largest error / tolerance ratio of one comparison (printed with -s); fails on a NaN or a ratio above 1."""
    ratio = (err / tol).max().item() if err.numel() else 0.0
    print(f"[ratio] {name}: {ratio:.3e}")
    assert not math.isnan(ratio), f"{name}: NaN (an element was not written)"
    assert ratio <= 1.0, f"{name}: error/tolerance {ratio:.3e}"
    return ratio


def _cdiv(a, b):
    return (a + b - 1) // b


def _stats_ppc(B, HW):
    """Pixels per CTA of gn_stats / ch_stats / gn_bwd_sums (stats_ppc in norm_elementwise.cu)."""
    ppc = 256
    while ppc > 8 and B * _cdiv(HW, ppc) < 592:
        ppc >>= 1
    return ppc


def _inputs(B, H, W, C1, C2, dc=False, seed=0):
    g = torch.Generator().manual_seed(seed)

    def mk(c):
        x = torch.randn(B, H, W, c, generator=g)
        return (x * 0.5 + 8.0 if dc else x).to(DEV)
    return mk(C1), (mk(C2) if C2 else None)


def _bank(B, C, seed, off=20, extra=44):
    """An emb / embz block [B][2C] (scale | shift) as a column block of a wider [B][ld] bank, ld > 2C, like the engine's
    Linear bank.  Returns (bank, view of the block, ld)."""
    g = torch.Generator().manual_seed(seed)
    ld = off + 2 * C + extra
    bank = (0.3 * torch.randn(B, ld, generator=g)).to(DEV)
    return bank, bank[:, off:off + 2 * C], ld


def _cat_nchw(x1, x2):
    x = x1 if x2 is None else torch.cat([x1, x2], dim=3)
    return x.double().permute(0, 3, 1, 2)


def _resample(h, rs):
    if rs == RESAMPLE_UP2:
        return F.interpolate(h, scale_factor=2, mode="nearest")
    if rs == RESAMPLE_DOWN2:
        return F.avg_pool2d(h, 2)
    return h


def _resample_t(g, rs):
    """Transpose of _resample applied to an NCHW gradient at the resampled size."""
    if rs == RESAMPLE_UP2:
        return F.avg_pool2d(g, 2) * 4.0
    if rs == RESAMPLE_DOWN2:
        return 0.25 * F.interpolate(g, scale_factor=2, mode="nearest")
    return g


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _exact_stats(x):
    """Exact per-(b, group) mean / var of an NCHW float64 tensor and the sums of |x| and x^2 the error bounds use."""
    B, C = x.shape[:2]
    xg = x.reshape(B, 32, -1)
    n = xg.shape[2]
    mean = xg.mean(2)
    var = (xg * xg).mean(2) - mean * mean
    return mean, var, xg.abs().sum(2), (xg * xg).sum(2), n


def _stat_error(x, nadd):
    """Bounds on the kernels' group mean, rstd (relative) given fp32 partial sums with at most `nadd` fp32 roundings on any
    path from an element to the fp64 group sum: |dS1| <= nadd*u*sum|x|, |dS2| <= nadd*u*sum x^2.  The variance is
    E[x^2] - mean^2 of those sums, so its error is the error of E[x^2] -- relative to E[x^2], not to the variance: a DC offset
    multiplies the relative error of rstd by (1 + mean^2/var) (257 for mean 8, std 0.5)."""
    mean, var, a1, a2, n = _exact_stats(x)
    dmean = nadd * U * a1 / n
    dvar = nadd * U * a2 / n + (2 * mean.abs() + dmean) * dmean
    rstd = 1.0 / torch.sqrt(var + EPS)
    rel_rstd = 0.5 * dvar / (var + EPS) + 3 * U      # first order in dvar; + rounding of rstd to fp32
    return mean, rstd, dmean, rel_rstd


def _per_channel(t, C):
    """[B][32] per-group values -> [B][C] per channel."""
    return t.repeat_interleave(C // 32, dim=1)


def _coef_ref(x, gamma, beta, emb, embz, nadd):
    """float64 ab rows [B][2][C] from the exact statistics and their tolerance for a kernel whose statistics have `nadd`
    fp32 roundings per element (see _stat_error)."""
    B, C = x.shape[:2]
    mean, rstd, dmean, rel_rstd = (_per_channel(t, C) for t in _stat_error(x, nadd))
    g, b = gamma.double()[None], beta.double()[None]
    a0 = g * rstd
    A, Bv = a0.clone(), b - mean * a0
    magB = b.abs() + (mean * a0).abs()
    sc = torch.ones_like(A)
    for v in (emb, embz):
        if v is not None:
            s, sh = 1.0 + v.double()[:, :C], v.double()[:, C:2 * C]
            A, Bv, magB, sc = A * s, Bv * s + sh, magB * s.abs() + sh.abs(), sc * s.abs()
    # a: gamma*rstd*s*zs -- rstd's error plus one rounding per product and per (1 + scale): 6u
    tolA = A.abs() * (rel_rstd + 6 * U)
    # b: the mean's error and rstd's through mean*a, then one rounding per op of ((beta - mean*a)*s + sh)*zs + zsh: 8u
    tolB = sc * ((mean * a0).abs() * rel_rstd + a0.abs() * dmean) + 8 * U * magB
    return torch.stack([A, Bv], 1), torch.stack([tolA, tolB], 1)


def _run_gn_stats(x1, x2, B, HW):
    C1, C2 = x1.shape[3], (x2.shape[3] if x2 is not None else 0)
    sums = _nan((B, 32, 2), torch.float64)
    _native.check(_L().pdae_gn_stats(_p(x1), C1, _p(x2), C2, B, HW, _p(sums), _stream()), "gn_stats")
    return sums


def _run_gn_coef(sums, gamma, beta, B, C, HW, emb, eld, embz, zld):
    ab = _nan((B, 2, C))
    _native.check(_L().pdae_gn_coef(_p(sums), _p(gamma), _p(beta), B, C, HW, EPS, _p(emb), eld, _p(embz), zld, _p(ab), _stream()),
                  "gn_coef")
    return ab


def _run_ch_stats(x, B, HW):
    C = x.shape[3]
    chs = _nan((B, C, 2))
    _native.check(_L().pdae_ch_stats(_p(x), B, HW, C, _p(chs), _stream()), "ch_stats")
    return chs


# ---- statistics and coefficients ------------------------------------------------------------------------------------
# (C1, C2, B, H, W, dc):  C = 32 with 4x4 images (8-pixel chunks), 96, 192 (L = 48: 16 idle threads per CTA), 512,
# 1024 (L = 256, the lane-layout limit) at B = 3 x 250 x 250 (256-pixel chunks, ragged tail); concats 64+32, 384+512 (a
# 28-channel group straddles the seam) and 512+512; a DC-offset input (mean 8, std 0.5).
STATS_SHAPES = [
    (32, 0, 2, 4, 4, False),
    (96, 0, 3, 17, 13, False),
    (192, 0, 2, 32, 32, False),
    (512, 0, 4, 16, 16, False),
    (1024, 0, 3, 250, 250, False),
    (64, 32, 2, 8, 8, False),
    (384, 512, 3, 64, 64, False),
    (512, 512, 3, 250, 250, False),
    (384, 512, 3, 64, 64, True),
]


@pytest.mark.parametrize("C1,C2,B,H,W,dc", STATS_SHAPES)
def test_gn_stats_and_ch_stats_match_float64(C1, C2, B, H, W, dc):
    HW = H * W
    x1, x2 = _inputs(B, H, W, C1, C2, dc, seed=C1 + C2 + H)
    ppc = _stats_ppc(B, HW)
    sums = _run_gn_stats(x1, x2, B, HW)
    chs = [_run_ch_stats(x, B, HW) for x in (x1, x2) if x is not None]
    torch.cuda.synchronize()
    x = _cat_nchw(x1, x2)
    C = C1 + C2
    xg = x.reshape(B, 32, -1)
    ref = torch.stack([xg.sum(2), (xg * xg).sum(2)], 2)
    mag = torch.stack([xg.abs().sum(2), (xg * xg).sum(2)], 2)
    # gn_stats: each thread sums its pixels of a chunk in fp32, the rows of a CTA meet by fp32 shared atomics: at most ppc
    # fp32 roundings per element before the fp64 group sums (+1 for the fma of x*x)
    tag = f"C={C1}+{C2} B={B} {H}x{W}{' dc' if dc else ''}"
    _report(f"gn_stats {tag}", (sums - ref).abs(), (ppc + 1) * U * mag + 1e-300)
    # ch_stats: the same per CTA, then one fp32 atomic per CTA into the per-channel total (cdiv(HW, ppc) more roundings)
    nadd = ppc + _cdiv(HW, ppc) + 1
    xs = [t for t in (x1, x2) if t is not None]
    for i, (t, c) in enumerate(zip(xs, chs)):
        td = t.double().reshape(B, HW, -1)
        r = torch.stack([td.sum(1), (td * td).sum(1)], 2)
        m = torch.stack([td.abs().sum(1), (td * td).sum(1)], 2)
        _report(f"ch_stats[{i}] {tag}", (c.double() - r).abs(), nadd * U * m + 1e-300)


COEF_CASES = [  # (C1, C2, B, H, W, dc, emb, embz)
    (32, 0, 2, 4, 4, False, False, False),
    (96, 0, 3, 17, 13, False, True, False),
    (192, 0, 2, 32, 32, False, True, True),
    (1024, 0, 3, 250, 250, False, True, True),
    (64, 32, 2, 8, 8, False, False, True),
    (384, 512, 3, 64, 64, False, True, True),
    (512, 512, 2, 32, 32, False, True, False),
    (384, 512, 3, 64, 64, True, True, True),
]


@pytest.mark.parametrize("C1,C2,B,H,W,dc,use_emb,use_embz", COEF_CASES)
def test_gn_coef_both_statistics_paths_match_float64(C1, C2, B, H, W, dc, use_emb, use_embz):
    """gn_stats -> gn_coef (fp32 mode) and ch_stats -> gn_coef_ch (the tensor-core mode's statistics form) against the
    float64 coefficients, and against each other; emb / embz are column blocks of a bank with ld > 2C."""
    C, HW = C1 + C2, H * W
    x1, x2 = _inputs(B, H, W, C1, C2, dc, seed=7 + C)
    g = torch.Generator().manual_seed(C)
    gamma = (1.0 + 0.3 * torch.randn(C, generator=g)).to(DEV)
    beta = (0.3 * torch.randn(C, generator=g)).to(DEV)
    _, emb, eld = _bank(B, C, 1) if use_emb else (None, None, 0)
    _, embz, zld = _bank(B, C, 2) if use_embz else (None, None, 0)
    sums = _run_gn_stats(x1, x2, B, HW)
    ab1 = _run_gn_coef(sums, gamma, beta, B, C, HW, emb, eld, embz, zld)
    chs1 = _run_ch_stats(x1, B, HW)
    chs2 = _run_ch_stats(x2, B, HW) if x2 is not None else None
    ab2 = _nan((B, 2, C))
    _native.check(_L().pdae_gn_coef_ch(_p(chs1), C1, _p(chs2), C2, _p(gamma), _p(beta), B, HW, EPS, _p(emb), eld, _p(embz), zld,
                                       _p(ab2), _stream()), "gn_coef_ch")
    torch.cuda.synchronize()
    x = _cat_nchw(x1, x2)
    ppc = _stats_ppc(B, HW)
    ref1, tol1 = _coef_ref(x, gamma, beta, emb, embz, ppc + 1)
    # ch_stats sums are fp32 totals (ppc + cdiv(HW, ppc) + 1 roundings), gn_coef_ch adds them per group in fp64
    ref2, tol2 = _coef_ref(x, gamma, beta, emb, embz, ppc + _cdiv(HW, ppc) + 2)
    tag = f"C={C1}+{C2} B={B} {H}x{W}{' dc' if dc else ''} emb={int(use_emb)} embz={int(use_embz)}"
    _report(f"gn_coef {tag}", (ab1.double() - ref1).abs(), tol1)
    _report(f"gn_coef_ch {tag}", (ab2.double() - ref2).abs(), tol2)
    _report(f"gn_coef vs gn_coef_ch {tag}", (ab1.double() - ab2.double()).abs(), tol1 + tol2)


# ---- forward apply --------------------------------------------------------------------------------------------------
# every (src1, src2, act, raw) dtype combination pdae_gn_apply accepts
APPLY_KEYS = [
    (PDAE_F32, PDAE_F32, PDAE_F32, PDAE_F32),
    (PDAE_F32, PDAE_F32, PDAE_BF16, PDAE_F32),
    (PDAE_F32, PDAE_F32, PDAE_BF16, PDAE_BF16),
    (PDAE_BF16, PDAE_F32, PDAE_BF16, PDAE_F32),
    (PDAE_BF16, PDAE_BF16, PDAE_BF16, PDAE_BF16),
    (PDAE_BF16, PDAE_F32, PDAE_BF16, PDAE_BF16),
    (PDAE_F32, PDAE_BF16, PDAE_BF16, PDAE_F32),
    (PDAE_F32, PDAE_BF16, PDAE_BF16, PDAE_BF16),
    (PDAE_BF16, PDAE_BF16, PDAE_BF16, PDAE_F32),
    (PDAE_BF16, PDAE_F32, PDAE_F32, PDAE_F32),
    (PDAE_BF16, PDAE_BF16, PDAE_F32, PDAE_F32),
    (PDAE_F32, PDAE_BF16, PDAE_F32, PDAE_F32),
]
# (C1, C2): 64 + 32 takes the 8-wide bf16 path for RESAMPLE_NONE, 36 + 28 (C1 % 8 != 0) the generic one, 64 alone has no
# second source
APPLY_CHANNELS = [(64, 32), (36, 28), (64, 0)]
TANH_APPROX_ERR = 2.0 ** -10.987     # PTX ISA: maximum error of tanh.approx.f32 over its whole range


def _ulp_bf16(v):
    """bf16 ulp of |v| (8 significant bits): 2^(e - 8) for v = m 2^e, m in [0.5, 1)."""
    _, e = torch.frexp(v)
    return torch.where(v != 0, torch.ldexp(torch.ones_like(v), e - 8), torch.full_like(v, 2.0 ** -133))


def _apply_ref(xs, ab, silu, rs, B, C):
    """float64 R(f(a*x + b)), the magnitude R(|a*x| + |b|) that bounds its fp32 evaluation error, and R(|a*x + b|/2) that
    scales the tanh.approx error of the fast SiLU (NCHW)."""
    x = _cat_nchw(*xs)
    if ab is None:
        a, b = torch.ones(B, C, 1, 1, dtype=torch.float64, device=DEV), torch.zeros(B, C, 1, 1, dtype=torch.float64, device=DEV)
    else:
        a, b = ab[:, 0].double()[:, :, None, None], ab[:, 1].double()[:, :, None, None]
    r = a * x + b
    mag = (a * x).abs() + b.abs()
    y = F.silu(r) if silu else r
    return _resample(y, rs), _resample(mag, rs), _resample(r.abs() * 0.5, rs)


def _raw_ref(xs, rs, raw_dt):
    """What out_raw must hold: the source values themselves (NONE / UP2, rounded to bf16 only if raw is bf16 and a source is
    fp32), or the fp32 2x2 mean ((x00 + x01) + x10) + x11 times 0.25 in the kernel's order (DOWN2)."""
    x = torch.cat([t.float() for t in xs if t is not None], dim=3)
    if rs == RESAMPLE_UP2:
        x = x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    elif rs == RESAMPLE_DOWN2:
        x = (((x[:, 0::2, 0::2] + x[:, 0::2, 1::2]) + x[:, 1::2, 0::2]) + x[:, 1::2, 1::2]) * 0.25
    return x.to(raw_dt)


def _out_hw(H, W, rs):
    return (2 * H, 2 * W) if rs == RESAMPLE_UP2 else ((H // 2, W // 2) if rs == RESAMPLE_DOWN2 else (H, W))


def _apply8_loops(C1, C2, HW):
    """Which loops of apply8_loop the 8-wide gn_apply launch runs for one image of HW pixels: (some thread runs the unrolled
    4-pixel body, some thread runs the scalar tail).  Mirrors the grid of pdae_gn_apply's fast branch (256 // (C/8) pixel
    rows per CTA, 8 pixels per thread, at most 148*16 CTAs per image) and the loop bounds with U = 4."""
    L8 = (C1 + C2) // 8
    ppc = 256 // L8
    stride = min(max(_cdiv(HW, ppc * 8), 1), 148 * 16) * ppc
    unrolled = tail = False
    for pix in range(min(stride, HW)):
        while pix + 3 * stride < HW:
            unrolled, pix = True, pix + 4 * stride
        tail = tail or pix < HW
    return unrolled, tail


@pytest.mark.parametrize("rs", [RESAMPLE_NONE, RESAMPLE_UP2, RESAMPLE_DOWN2], ids=RS_NAMES.get)
@pytest.mark.parametrize("key", APPLY_KEYS, ids=lambda k: "".join("fb"[d] for d in k))
def test_gn_apply_matches_float64(key, rs):
    # 6x10: every pixel of the 8-wide path goes through its scalar tail loop; 40x41 (40x42 for DOWN2, which needs even
    # sizes): several pixel strides per thread, so the unrolled body runs and a ragged remainder is left for the tail
    for B, H, W in ((2, 6, 10), (2, 40, 42 if rs == RESAMPLE_DOWN2 else 41)):
        _apply_case(key, rs, B, H, W)


def _apply_case(key, rs, B, H, W):
    d1, d2, da, dr = key
    worst = 0.0
    for C1, C2 in APPLY_CHANNELS:
        C = C1 + C2
        x1, x2 = _inputs(B, H, W, C1, C2, seed=C1)
        s1 = x1.to(DT[d1])
        s2 = x2.to(DT[d2]) if x2 is not None else None
        g = torch.Generator().manual_seed(C)
        ab_t = torch.stack([1.0 + 0.5 * torch.randn(B, C, generator=g), 0.5 * torch.randn(B, C, generator=g)], 1).to(DEV)
        Ho, Wo = _out_hw(H, W, rs)
        fast = rs == RESAMPLE_NONE and da == PDAE_BF16 and C1 % 8 == 0 and C2 % 8 == 0
        if fast and H * W > 1000:
            assert _apply8_loops(C1, C2, H * W) == (True, True), "the large image no longer runs both loops of apply8_loop"
        for silu in (0, 1):
            for ab in (None, ab_t):
                with_raw = not (silu and ab is None)     # one combination with out_raw = NULL
                act = _nan((B, Ho, Wo, C), DT[da])
                raw = _nan((B, Ho, Wo, C), DT[dr]) if with_raw else None
                _native.check(_L().pdae_gn_apply(_p(s1), d1, C1, _p(s2), d2, C2, _p(ab), silu, rs, B, H, W, _p(act), da, _p(raw),
                                                 dr, _stream()), "gn_apply")
                torch.cuda.synchronize()
                ref, mag, half_r = _apply_ref((s1, s2), ab, silu, rs, B, C)
                ref, mag, half_r = _nhwc(ref), _nhwc(mag), _nhwc(half_r)
                # fp32 evaluation: one rounding in the fma, SiLU x/(1+expf(-x)) within a few ulps, the 2x2 sum and mean of
                # DOWN2: 16u of the magnitudes is a bound with margin
                e32 = 16 * U * mag
                if silu and fast:   # h + h*tanh.approx(h), h = x/2: |h| times the tanh.approx error
                    e32 = e32 + TANH_APPROX_ERR * half_r
                tol = e32 if da == PDAE_F32 else 0.5 * _ulp_bf16(ref.abs() + e32) + e32   # + half a bf16 ulp from the rounding
                tag = (f"gn_apply {''.join('fb'[d] for d in key)} {RS_NAMES[rs]} {H}x{W} C={C1}+{C2} silu={silu} "
                       f"ab={'y' if ab is not None else 'n'}{' 8-wide' if fast else ''}")
                worst = max(worst, _report(tag, (act.double() - ref).abs(), tol + 1e-300))
                if with_raw:
                    rr = _raw_ref((s1, s2), rs, DT[dr])
                    assert torch.equal(raw.view(torch.int16) if dr == PDAE_BF16 else raw.view(torch.int32),
                                       rr.view(torch.int16) if dr == PDAE_BF16 else rr.view(torch.int32)), f"{tag}: raw output"
    print(f"[ratio] gn_apply {key} {RS_NAMES[rs]} {H}x{W} worst: {worst:.3e}")


@pytest.mark.parametrize("key", [(0, 0, 0, 1), (1, 0, 0, 1), (0, 1, 0, 1), (1, 1, 0, 1), (2, 0, 1, 0), (0, 0, 3, 0)])
def test_gn_apply_rejects_unsupported_dtypes_and_launches_nothing(key):
    d1, d2, da, dr = key
    B, H, W, C1, C2 = 2, 4, 4, 32, 32
    s1 = torch.zeros(B, H, W, C1, device=DEV)
    s2 = torch.zeros(B, H, W, C2, device=DEV)
    act = _nan((B, H, W, C1 + C2))
    raw = _nan((B, H, W, C1 + C2))
    rc = _L().pdae_gn_apply(_p(s1), d1, C1, _p(s2), d2, C2, None, 0, RESAMPLE_NONE, B, H, W, _p(act), da, _p(raw), dr, _stream())
    torch.cuda.synchronize()
    assert rc != 0 and b"unsupported dtype" in _L().pdae_last_error()
    assert torch.isnan(act).all() and torch.isnan(raw).all()


@pytest.mark.parametrize("rs", [RESAMPLE_NONE, RESAMPLE_UP2, RESAMPLE_DOWN2], ids=RS_NAMES.get)
@pytest.mark.parametrize("raw_dt", [PDAE_F32, PDAE_BF16], ids=["raw_f32", "raw_split"])
def test_gn_apply_split3_matches_float64(rs, raw_dt):
    B, H, W = 2, 6, 10
    for C1, C2 in ((64, 32), (36, 28), (96, 0)):
        C = C1 + C2
        x1, x2 = _inputs(B, H, W, C1, C2, seed=3 + C1)
        g = torch.Generator().manual_seed(C)
        ab_t = torch.stack([1.0 + 0.5 * torch.randn(B, C, generator=g), 0.5 * torch.randn(B, C, generator=g)], 1).to(DEV)
        Ho, Wo = _out_hw(H, W, rs)
        for silu in (0, 1):
            for ab in (None, ab_t):
                act3 = _nan((B, Ho, Wo, 3 * C), torch.bfloat16)
                raw = _nan((B, Ho, Wo, 3 * C), torch.bfloat16) if raw_dt == PDAE_BF16 else _nan((B, Ho, Wo, C))
                _native.check(_L().pdae_gn_apply_split3(_p(x1), C1, _p(x2), C2, _p(ab), silu, rs, B, H, W, _p(act3), _p(raw),
                                                        raw_dt, _stream()), "gn_apply_split3")
                torch.cuda.synchronize()
                tag = f"gn_apply_split3 {RS_NAMES[rs]} C={C1}+{C2} silu={silu} ab={'y' if ab is not None else 'n'}"
                hi, lo, hi2 = act3[..., :C], act3[..., C:2 * C], act3[..., 2 * C:]
                assert torch.equal(hi.view(torch.int16), hi2.view(torch.int16)), f"{tag}: third block != first"
                hif, lof = hi.float(), lo.float()
                # hi = bf16_rn(r) of the fp32 value r and lo = bf16_rn(r - hi): |lo| <= half an ulp of hi, and hi is within
                # half a bf16 ulp (+ the fp32 evaluation error of r) of the float64 value
                assert bool((lof.abs() <= 0.5 * _ulp_bf16(hif.double()).float()).all()), f"{tag}: |lo| > ulp(hi)/2"
                ref, mag, _ = _apply_ref((x1, x2), ab, silu, rs, B, C)
                ref, mag = _nhwc(ref), _nhwc(mag)
                e32 = 16 * U * mag
                _report(f"{tag} hi", (hif.double() - ref).abs(), 0.5 * _ulp_bf16(ref.abs() + e32) + e32 + 1e-300)
                # lo keeps 8 more bits: |hi + lo - r| <= 2^-17 |r|; plus the fp32 evaluation of r (as for gn_apply)
                tol = 2.0 ** -16 * ref.abs() + 16 * U * mag * (1 + 2.0 ** -8)
                _report(tag, (hif.double() + lof.double() - ref).abs(), tol + 1e-300)
                rr = _raw_ref((x1, x2), rs, torch.float32)
                if raw_dt == PDAE_F32:
                    assert torch.equal(raw.view(torch.int32), rr.view(torch.int32)), f"{tag}: raw output"
                else:
                    rhi = rr.to(torch.bfloat16)
                    rlo = (rr - rhi.float()).to(torch.bfloat16)
                    want = torch.cat([rhi, rlo, rhi], dim=3)
                    assert torch.equal(raw.view(torch.int16), want.view(torch.int16)), f"{tag}: split raw output"


# ---- backward -------------------------------------------------------------------------------------------------------
BWD_CASES = [  # (C1, C2, B, H, W, rs, silu, emb, add, dx2, dc)
    (32, 0, 2, 4, 4, RESAMPLE_NONE, 1, False, False, False, False),
    (96, 0, 3, 18, 14, RESAMPLE_NONE, 1, True, True, False, False),
    (192, 0, 3, 16, 16, RESAMPLE_DOWN2, 1, False, True, False, False),
    (64, 32, 3, 8, 8, RESAMPLE_UP2, 1, True, True, True, False),
    (384, 512, 3, 32, 32, RESAMPLE_NONE, 1, True, False, True, False),
    (512, 512, 3, 64, 64, RESAMPLE_DOWN2, 0, False, True, True, False),
    (384, 512, 2, 16, 16, RESAMPLE_UP2, 0, True, True, False, False),
    (1024, 0, 3, 160, 161, RESAMPLE_NONE, 1, True, True, False, False),   # L = 256; 128-pixel chunks, ragged tail of 32
    (512, 0, 3, 64, 64, RESAMPLE_NONE, 1, True, True, False, True),
    (384, 512, 3, 32, 32, RESAMPLE_DOWN2, 1, True, True, True, True),
]


def _bwd_id(c):
    C1, C2, B, H, W, rs, silu, emb, add, dx2, dc = c
    return (f"{C1}+{C2}-b{B}-{H}x{W}-{RS_NAMES[rs]}-silu{silu}" + ("-emb" if emb else "") + ("-add" if add else "")
            + ("-dx2" if dx2 else "") + ("-dc" if dc else ""))


@pytest.mark.parametrize("C1,C2,B,H,W,rs,silu,use_emb,use_add,want_dx2,dc", BWD_CASES, ids=[_bwd_id(c) for c in BWD_CASES])
def test_gn_backward_three_passes_match_float64_autograd(C1, C2, B, H, W, rs, silu, use_emb, use_add, want_dx2, dc):
    C, HW = C1 + C2, H * W
    Ho, Wo = _out_hw(H, W, rs)
    x1, x2 = _inputs(B, H, W, C1, C2, dc, seed=11 + C + H)
    g = torch.Generator().manual_seed(3 * C + 1)
    gamma = (1.0 + 0.3 * torch.randn(C, generator=g)).to(DEV)
    beta = (0.3 * torch.randn(C, generator=g)).to(DEV)
    dy = torch.randn(B, Ho, Wo, C, generator=g).to(DEV)
    add_ld = C + 12
    add = torch.randn(B, Ho, Wo, add_ld, generator=g).to(DEV) if use_add else None
    dg0 = torch.randn(C, generator=g).to(DEV)             # dgamma / dbeta accumulate into what is there
    db0 = torch.randn(C, generator=g).to(DEV)
    _, emb, eld = _bank(B, C, 5) if use_emb else (None, None, 0)
    _, embz, zld = _bank(B, C, 6) if use_emb else (None, None, 0)
    if use_emb:
        dbank_e, dbank_z = _nan((B, eld)), _nan((B, zld))
        demb, dembz = dbank_e[:, 20:20 + 2 * C], dbank_z[:, 20:20 + 2 * C]
    else:
        dbank_e = dbank_z = demb = dembz = None
    # forward coefficients and statistics as the training forward leaves them
    sums = _run_gn_stats(x1, x2, B, HW)
    ab = _run_gn_coef(sums, gamma, beta, B, C, HW, emb, eld, embz, zld)
    L = _L()
    S = _nan((B, C, 2))
    kk = _nan((B, 3, C))
    dgamma, dbeta = dg0.clone(), db0.clone()
    dx1 = _nan((B, H, W, C1))
    dx2 = _nan((B, H, W, C2)) if want_dx2 else None
    _native.check(L.pdae_gn_bwd_sums(_p(x1), C1, _p(x2), C2, _p(ab), _p(dy), silu, rs, B, H, W, _p(S), _stream()), "gn_bwd_sums")
    _native.check(L.pdae_gn_bwd_coef(_p(S), _p(sums), _p(gamma), _p(beta), _p(emb), eld, _p(embz), zld, B, C, HW, EPS, _p(kk),
                                     _p(dgamma), _p(dbeta), _p(demb), eld, _p(dembz), zld, _stream()), "gn_bwd_coef")
    _native.check(L.pdae_gn_bwd_apply(_p(x1), C1, _p(x2), C2, _p(ab), _p(kk), _p(dy), silu, rs, B, H, W, _p(add), add_ld,
                                      _p(dx1), _p(dx2), _stream()), "gn_bwd_apply")
    torch.cuda.synchronize()

    # float64 autograd of the forward graph
    x = _cat_nchw(x1, x2).requires_grad_()
    gam, bet = gamma.double().requires_grad_(), beta.double().requires_grad_()
    e = emb.double().requires_grad_() if use_emb else None
    z = embz.double().requires_grad_() if use_emb else None
    h = F.group_norm(x, 32, gam, bet, eps=EPS)
    u = h
    for v in (e, z):
        if v is not None:
            u = u * (1.0 + v[:, :C, None, None]) + v[:, C:, None, None]
    y = _resample(F.silu(u) if silu else u, rs)
    loss = (y * dy.double().permute(0, 3, 1, 2)).sum()
    if use_add:   # the skip path: R(x) meets the add gradient
        loss = loss + (_resample(x, rs) * add[..., :C].double().permute(0, 3, 1, 2)).sum()
    loss.backward()
    ud, xd = u.detach(), x.detach()
    del h, u, y, loss          # the reference is only needed through x.grad / e.grad / z.grad from here on

    # ---- error bounds (float64, per element / per channel; full-size temporaries are freed once reduced) ----
    ppc = _stats_ppc(B, HW)
    mean, rstd, dmean, rel_rstd = (_per_channel(t, C)[:, :, None, None] for t in _stat_error(xd, ppc + 1))
    e4 = lambda t: t[:, :, None, None]                                          # noqa: E731
    g_rt = _resample_t(dy.double().permute(0, 3, 1, 2), rs)          # R^T(dy)
    g_abs = _resample_t(dy.double().abs().permute(0, 3, 1, 2), rs)
    gather_err = (3 * U * g_abs) if rs == RESAMPLE_UP2 else 0.0     # the four-term fp32 sum of UP2
    if silu:
        sg = torch.sigmoid(ud)
        dsl = sg * (1 + ud * (1 - sg))
        du = g_rt * dsl
        # the kernel's pre-activation fma(a, x, b) uses the fp32 ab rows (their gn_coef error bound) plus one rounding;
        # |silu''| <= 0.5; dsilu(u) with expf and three more roundings is within 8u(1 + |u|)
        _, tol_ab = _coef_ref(xd, gamma, beta, emb, embz, ppc + 1)
        du_pre = xd.abs() * e4(tol_ab[:, 0]) + e4(tol_ab[:, 1]) + U * ud.abs()
        ddu = g_abs * (0.5 * du_pre + 8 * U * (1 + ud.abs())) + gather_err * dsl.abs() + U * du.abs()
        del sg, dsl, du_pre
    else:
        du = g_rt
        ddu = gather_err if rs == RESAMPLE_UP2 else torch.zeros_like(du)
    del ud, g_rt, g_abs, gather_err
    nb = ppc + _cdiv(HW, ppc) + 2        # fp32 roundings per term of S: per-thread chain and shared atomics, global atomics
    S1, S2 = du.sum((2, 3)), (du * xd).sum((2, 3))
    dS1 = nb * U * du.abs().sum((2, 3)) + ddu.sum((2, 3))
    dS2 = (nb + 1) * U * (du * xd).abs().sum((2, 3)) + (ddu * xd.abs()).sum((2, 3))
    m2, r2, dm2, rr2 = (t[:, :, 0, 0] for t in (mean, rstd, dmean, rel_rstd))
    dbt, dgt = S1, r2 * (S2 - m2 * S1)
    ddbt = dS1
    # dgt = rstd (S2 - mean S1) in fp64 from the fp32 S: the sums' errors, mean's and rstd's errors.  With a DC offset
    # S2 ~ mean S1 cancels and mean * dS1 dominates.
    ddgt = r2 * (dS2 + m2.abs() * dS1 + dm2 * S1.abs()) + rr2 * dgt.abs()
    s = (1.0 + emb.double()[:, :C]) if use_emb else torch.ones_like(dbt)
    sh = emb.double()[:, C:] if use_emb else torch.zeros_like(dbt)
    zs = (1.0 + embz.double()[:, :C]) if use_emb else torch.ones_like(dbt)
    gd, bd = gamma.double()[None], beta.double()[None]
    gt = gd * s * zs
    cpg, n = C // 32, HW * (C // 32)
    grp = lambda t: t.reshape(B, 32, cpg).sum(2).repeat_interleave(cpg, 1)     # noqa: E731
    gA, gB = grp(gt * dbt), grp(gt * dgt)
    dgA = grp(gt.abs() * ddbt + 4 * U * (gt * dbt).abs())
    dgB = grp(gt.abs() * ddgt + 4 * U * (gt * dgt).abs())
    k0, k1 = r2 * gt, -r2 * r2 * gB / n
    dk0 = k0.abs() * (rr2 + 6 * U)
    dk1 = r2 * r2 / n * dgB + k1.abs() * (2 * rr2 + 2 * U)
    t2 = (r2 * gA / n).abs()
    k2 = -r2 * gA / n - k1 * m2
    dk2 = r2 / n * dgA + t2 * (rr2 + 2 * U) + dk1 * m2.abs() + k1.abs() * dm2 + 2 * U * (t2 + (k1 * m2).abs())
    # dx = k0 du + k1 x + k2 in two fmas (+ R^T(add), one more rounding and the UP2 four-term sum)
    tdx = (e4(dk0) * du.abs() + e4(k0.abs()) * ddu + e4(dk1) * xd.abs() + e4(dk2)
           + 2 * U * (e4(k0.abs()) * du.abs() + e4(k1.abs()) * xd.abs() + e4(k2.abs())))
    if use_add:
        a_abs = _resample_t(add[..., :C].double().abs().permute(0, 3, 1, 2), rs)
        tdx = tdx + U * (x.grad.abs() + a_abs) + (3 * U * a_abs if rs == RESAMPLE_UP2 else 0.0)
    tdx = _nhwc(tdx)
    ref_dx = _nhwc(x.grad)
    tag = _bwd_id((C1, C2, B, H, W, rs, silu, use_emb, use_add, want_dx2, dc))
    _report(f"gn_bwd dx1 {tag}", (dx1.double() - ref_dx[..., :C1]).abs(), tdx[..., :C1] + 1e-300)
    if want_dx2:
        _report(f"gn_bwd dx2 {tag}", (dx2.double() - ref_dx[..., C1:]).abs(), tdx[..., C1:] + 1e-300)
    # dgamma / dbeta: sum over b of dgt*s*zs (dbt*s*zs), fp32 atomics over B onto the prefilled values
    sz = (s * zs).abs()
    for name, got, base, grad, v, dv in (("dgamma", dgamma, dg0, gam.grad, dgt, ddgt), ("dbeta", dbeta, db0, bet.grad, dbt, ddbt)):
        terms = (v * s * zs).abs().sum(0)
        tol = (dv * sz + 4 * U * (v * s * zs).abs()).sum(0) + (B + 1) * U * (terms + base.double().abs())
        _report(f"gn_bwd {name} {tag}", (got.double() - base.double() - grad).abs(), tol)
    if use_emb:
        t_es = (ddgt * gd.abs() + ddbt * bd.abs()) * zs.abs() + 4 * U * ((dgt * gd).abs() + (dbt * bd).abs()) * zs.abs()
        t_esh = ddbt * zs.abs() + 2 * U * (dbt * zs).abs()
        t_zs = ddgt * (gd * s).abs() + ddbt * (bd * s + sh).abs() + 5 * U * ((dgt * gd * s).abs() + dbt.abs() * ((bd * s).abs() + sh.abs()))
        t_zsh = ddbt + U * dbt.abs()
        _report(f"gn_bwd demb {tag}", (demb.double() - e.grad).abs(), torch.cat([t_es, t_esh], 1))
        _report(f"gn_bwd dembz {tag}", (dembz.double() - z.grad).abs(), torch.cat([t_zs, t_zsh], 1))
        for bank in (dbank_e, dbank_z):   # nothing outside the (scale | shift) block is written
            assert torch.isnan(bank[:, :20]).all() and torch.isnan(bank[:, 20 + 2 * C:]).all(), f"{tag}: write outside demb block"
