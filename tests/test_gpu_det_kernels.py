"""The deterministic (DET) kernels through the C-ABI, each against float64 torch on the device and against its atomic twin.

DET kernels use no float atomics: every partial result is stored in its own slot of a caller-owned workspace and the slots are
summed in a fixed order.  Every case goes through one harness (_det_run), which checks what the model-level determinism tests
cannot see:
  - outputs and the workspace are filled with NaN (0xFFFF for bf16) before the launch, so an output that is added to instead of
    written, or a slot that is read but never written, shows up as a NaN;
  - the workspace is exactly *_workspace_bytes bytes at the start of a larger allocation, followed by a 4 KiB guard band of
    a sentinel byte that must be unchanged afterwards (an overrun lands in the data, it never faults);
  - one call with `need - 8` bytes must return PDAE_EINVAL and launch nothing (each entry point checks the size first);
  - a second run, with no zeroing in between, must give identical bits.
Tolerances are worst-case bounds of the kernels' arithmetic evaluated per element in float64 (u = 2^-24 per fp32 rounding; a
sum of n terms in any order is off by at most (n - 1) u sum|terms|; a wgmma fp32 accumulation step is counted as 2u, since the
tensor cores may truncate); _report prints the worst err / tol ratio of each comparison."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from pdae_b200 import _native
from pdae_b200._native import PDAE_BF16, PDAE_F32, RESAMPLE_DOWN2, RESAMPLE_NONE, RESAMPLE_UP2
from tests.test_gpu_conv_tc3 import _run as _tc3_run
from tests.test_gpu_norm_kernels import (EPS, RS_NAMES, U, _bank, _cat_nchw, _cdiv, _inputs, _nan, _nhwc, _out_hw, _p, _report,
                                         _resample_t, _stat_error, _stats_ppc, _stream, _ulp_bf16)
from tests.test_gpu_wgrad_tc import _split3, wgrad_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
PDAE_EINVAL = -1
GUARD = 4096
SENTINEL = 0x5A
U53 = 2.0 ** -53
BITS = {torch.float32: torch.int32, torch.float64: torch.int64, torch.bfloat16: torch.int16}


def _L():
    return _native.lib()


def _bits(t):
    return t.view(BITS[t.dtype])


def _fill_nan(t):
    if t.dtype == torch.bfloat16:
        t.view(torch.int16).fill_(-1)
    else:
        t.fill_(float("nan"))


class _Workspace:
    """`need` bytes of 0xFF (a NaN in fp32 and fp64) at the start of an allocation, then GUARD bytes of SENTINEL."""

    def __init__(self, need):
        assert need >= 0, f"workspace size query failed: {need} ({_L().pdae_last_error()})"
        self.need = int(need)
        self.buf = torch.full((self.need + GUARD,), SENTINEL, dtype=torch.uint8, device=DEV)
        self.buf[:self.need] = 0xFF
        self.ptr = ctypes.c_void_p(self.buf.data_ptr())

    def check_guard(self, tag):
        torch.cuda.synchronize()
        bad = (self.buf[self.need:] != SENTINEL).nonzero()
        assert bad.numel() == 0, f"{tag}: {bad.numel()} guard bytes past the {self.need}-byte workspace were written " \
                                 f"(first at +{bad[0].item()})"


def _det_run(tag, need, outs, run, arm=None, prefill=True, repeat=True):
    """The checks every DET case goes through.  run(ptr, nbytes) launches the DET entry point (or a plan's run, which ignores
    the arguments, when arm(ptr, nbytes) is the plan's set_deterministic).  Returns clones of `outs` after the first run."""
    ws = _Workspace(need)
    if prefill:
        for o in outs:
            _fill_nan(o)
    if need >= 8:
        before = [_bits(o).clone() for o in outs]
        rc = (arm or run)(ws.ptr, need - 8)
        torch.cuda.synchronize()
        assert rc == PDAE_EINVAL, f"{tag}: a workspace of need - 8 = {need - 8} bytes returned {rc}, not PDAE_EINVAL"
        assert all(torch.equal(_bits(o), b) for o, b in zip(outs, before)), f"{tag}: the rejected call wrote an output"
        assert bool((ws.buf[:need] == 0xFF).all()), f"{tag}: the rejected call wrote the workspace"
    if arm is not None:
        _native.check(arm(ws.ptr, need), f"{tag}: set_deterministic")
    _native.check(run(ws.ptr, need), tag)
    torch.cuda.synchronize()
    first = [o.clone() for o in outs]
    ws.check_guard(tag)
    if repeat:
        _native.check(run(ws.ptr, need), f"{tag} (repeat)")
        torch.cuda.synchronize()
        for i, (a, o) in enumerate(zip(first, outs)):
            assert torch.equal(_bits(a), _bits(o)), f"{tag}: output {i} differs between two runs with no zeroing in between"
        ws.check_guard(f"{tag} (repeat)")
    return first


def _assert_bitwise(tag, a, b):
    same = _bits(a) == _bits(b)
    assert bool(same.all()), f"{tag}: {int((~same).sum())} of {same.numel()} elements differ from the default kernel"
    print(f"[ratio] {tag}: bitwise equal")


def _batch_invariance(tag, make, run):
    """make(i) -> the inputs of image i (tensors with a leading batch dim of 1); run(inputs) -> per-image outputs (leading dim
    B).  Image 0 alone, at positions 0 and 4 of a batch of 5 and at position 1 of a batch of 3 must give identical bits."""
    x, o = make(0), [make(i) for i in range(1, 5)]
    cat = lambda items: tuple(torch.cat(parts) for parts in zip(*items))       # noqa: E731
    ref = None
    for items, pos in (([x], 0), ([x] + o, 0), (o + [x], 4), ([o[0], x, o[1]], 1)):
        got = [_bits(t[pos]).clone() for t in run(cat(items))]
        if ref is None:
            ref = got
        else:
            for i, (a, b) in enumerate(zip(ref, got)):
                assert torch.equal(a, b), f"{tag}: output {i} of the image at position {pos} of a batch of {len(items)} differs"
    print(f"[ratio] {tag}: batch invariant")


def _sum_tol(nadd, mag, extra=0.0):
    return nadd * U * mag + extra + 1e-300


# ---- ch_stats_det / gn_stats_det --------------------------------------------------------------------------------------
def _stats_ppc_det(HW):
    """stats_ppc_det (norm_elementwise.cu): pixels per CTA of ch_parts_kernel, from the image size alone."""
    ppc = 256
    while ppc > 8 and _cdiv(HW, ppc) < 16:
        ppc >>= 1
    return ppc


def _parts_roundings(C, HW):
    """fp32 roundings per element in ch_parts_kernel's partials: a thread's chain over its pixels, then the R pixel rows of
    the CTA in order.  Returns (that count, P = CTAs per image)."""
    ppc = _stats_ppc_det(HW)
    R = 256 // min(C // 4, 256)
    return _cdiv(ppc, R) + R + 1, _cdiv(HW, ppc)


def _run_stats_det(x1, x2, B, HW, tag):
    C1, C2 = x1.shape[3], (x2.shape[3] if x2 is not None else 0)
    need = _L().pdae_stats_det_workspace_bytes(B, HW, C1 + C2)
    ppc = _stats_ppc_det(HW)
    assert need == B * _cdiv(HW, ppc) * (C1 + C2) * 8, need
    sums = torch.empty(B, 32, 2, dtype=torch.float64, device=DEV)
    (sums,) = _det_run(f"gn_stats_det {tag}", need, [sums], lambda w, n: _L().pdae_gn_stats_det(
        _p(x1), C1, _p(x2), C2, B, HW, _p(sums), w, n, _stream()))
    chs = []
    for i, x in enumerate(t for t in (x1, x2) if t is not None):
        C = x.shape[3]
        c = torch.empty(B, C, 2, device=DEV)
        nb = _L().pdae_stats_det_workspace_bytes(B, HW, C)
        chs += _det_run(f"ch_stats_det[{i}] {tag}", nb, [c], lambda w, n, x=x, C=C, c=c: _L().pdae_ch_stats_det(
            _p(x), B, HW, C, _p(c), w, n, _stream()))
    return sums, chs


STATS_CASES = [  # (C1, C2, B, H, W, dc)
    (32, 0, 3, 4, 4, False),        # HW = 16: two 8-pixel CTAs; C = 32: 8 lanes, 32 pixel rows per CTA
    (96, 0, 2, 8, 8, False),        # HW = 64; L = 24: 10 rows of 24 lanes, 16 idle threads
    (1024, 0, 2, 16, 16, False),    # HW = 256: 16 CTAs of 16 pixels; L = 256, one row
    (6144, 0, 2, 8, 8, False),      # the channel limit: 48 KiB of shared memory, six quads per thread
    (96, 0, 2, 250, 250, False),    # 245 CTAs of 256 pixels, the last one ragged (36)
    (1024, 0, 1, 250, 250, False),
    (40, 56, 2, 8, 8, False),       # concat: group 13 (channels 39..41) straddles the seam
    (384, 512, 2, 16, 16, True),    # DC offset (mean 8, std 0.5)
]


@pytest.mark.parametrize("C1,C2,B,H,W,dc", STATS_CASES)
def test_stats_det_match_float64_and_the_atomic_kernels(C1, C2, B, H, W, dc):
    HW, C = H * W, C1 + C2
    tag = f"C={C1}+{C2} B={B} {H}x{W}{' dc' if dc else ''}"
    x1, x2 = _inputs(B, H, W, C1, C2, dc, seed=C + H)
    sums, chs = _run_stats_det(x1, x2, B, HW, tag)
    n32, P = _parts_roundings(C, HW)
    # ch_stats_det: the partials (n32 roundings), then stat_parts_reduce: lane r adds partials r, r + 8, ... in order and the
    # eight lane sums are added in order
    nch = n32 + _cdiv(P, 8) + 8
    xs = [t for t in (x1, x2) if t is not None]
    ppc_a = _stats_ppc(B, HW)
    for i, (t, c) in enumerate(zip(xs, chs)):
        td = t.double().reshape(B, HW, -1)
        ref = torch.stack([td.sum(1), (td * td).sum(1)], 2)
        mag = torch.stack([td.abs().sum(1), (td * td).sum(1)], 2)
        _report(f"ch_stats_det[{i}] {tag}", (c.double() - ref).abs(), _sum_tol(nch, mag))
        a = torch.zeros_like(c)
        _native.check(_L().pdae_ch_stats(_p(t), B, HW, t.shape[3], _p(a), _stream()), "ch_stats")
        torch.cuda.synchronize()
        # the atomic kernel: ppc_a + cdiv(HW, ppc_a) + 1 roundings (test_gpu_norm_kernels)
        _report(f"ch_stats_det vs ch_stats[{i}] {tag}", (c.double() - a.double()).abs(),
                _sum_tol(nch + ppc_a + _cdiv(HW, ppc_a) + 1, mag))
    x = _cat_nchw(x1, x2)
    xg = x.reshape(B, 32, -1)
    ref = torch.stack([xg.sum(2), (xg * xg).sum(2)], 2)
    mag = torch.stack([xg.abs().sum(2), (xg * xg).sum(2)], 2)
    # gn_stats_det: fp32 partials, then fp64 sums of P * C/32 terms (gn_group_reduce_kernel)
    f64 = (P * (C // 32) + 4) * U53 * mag
    _report(f"gn_stats_det {tag}", (sums - ref).abs(), _sum_tol(n32, mag, f64))
    sums_a = torch.zeros(B, 32, 2, dtype=torch.float64, device=DEV)
    _native.check(_L().pdae_gn_stats(_p(x1), C1, _p(x2), C2, B, HW, _p(sums_a), _stream()), "gn_stats")
    torch.cuda.synchronize()
    _report(f"gn_stats_det vs gn_stats {tag}", (sums - sums_a).abs(), _sum_tol(n32 + ppc_a + 1, mag, 2 * f64))
    if dc:
        # The variance E[x^2] - mean^2 formed from these sums carries their error relative to E[x^2], not to the variance:
        # with mean 8 and std 0.5 that multiplies its relative bound by 1 + mean^2 / var = 257.
        mean, var = xg.mean(2), xg.var(2, unbiased=False)
        amp = (1 + mean * mean / var).mean().item()
        print(f"[ratio] DC offset: variance error amplification {amp:.1f}")
        assert 240 < amp < 275, amp
        _, _, _, rel_rstd = _stat_error(x, n32 + 1)
        n = HW * (C // 32)
        var_k = sums[..., 1] / n - (sums[..., 0] / n) ** 2
        _report(f"gn_stats_det variance {tag}", (var_k - var).abs(), 2 * rel_rstd * (var + EPS))
    if H <= 16:
        def run(xb):
            s, c = _run_stats_det(xb[0], xb[1] if C2 else None, xb[0].shape[0], HW, f"{tag} batch")
            return [s] + c
        _batch_invariance(f"stats_det {tag}", lambda i: tuple(t for t in _inputs(1, H, W, C1, C2, dc, seed=50 + i) if t is not None),
                          run)


# ---- stem det ---------------------------------------------------------------------------------------------------------
def _stem_grid_x(H, W, Cout, stride):
    Ho, Wo, ppc = H // stride, W // stride, 256 // (Cout // 8)
    return max(min(_cdiv(Ho * (Wo // 4), ppc * 2), 148 * 8), 1)


def _stem_inputs(B, Cin, H, W, Cout, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, H, W, generator=g).to(DEV)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (3 * Cin ** 0.5)).to(DEV)
    b = (0.3 * torch.randn(Cout, generator=g)).to(DEV)
    return x, w, b


def _stem_det(x, wp, b, Cout, stride, tag):
    B, Cin, H, W = x.shape
    out = torch.empty(B, H // stride, W // stride, Cout, dtype=torch.bfloat16, device=DEV)
    st = torch.empty(B, Cout, 2, device=DEV)
    need = _L().pdae_stem_conv_det_workspace_bytes(B, H, W, Cout, stride)
    assert need == B * _stem_grid_x(H, W, Cout, stride) * Cout * 8, need
    return _det_run(tag, need, [out, st], lambda w, n: _L().pdae_stem_conv_bf16_det(
        _p(x), _p(wp), _p(b), _p(out), _p(st), B, H, W, Cin, Cout, stride, w, n, _stream()))


STEM_CASES = [  # (B, Cin, H, W, Cout, stride)
    (2, 1, 8, 8, 8, 1),
    (3, 2, 16, 12, 64, 1),
    (2, 3, 32, 32, 256, 1),
    (2, 4, 16, 16, 128, 1),
    (1, 3, 288, 288, 256, 1),     # the grid reaches its 148 x 8 cap: the grid-stride loop runs
    (2, 3, 32, 32, 64, 2),
    (2, 1, 16, 24, 8, 2),
    (3, 4, 16, 16, 128, 2),
]


@pytest.mark.parametrize("B,Cin,H,W,Cout,stride", STEM_CASES)
def test_stem_det_matches_float64_and_the_default_stem(B, Cin, H, W, Cout, stride):
    tag = f"stem_det B={B} Cin={Cin} {H}x{W} Cout={Cout} s={stride}"
    x, w, b = _stem_inputs(B, Cin, H, W, Cout, seed=Cin + Cout + H)
    wp = w.reshape(Cout, Cin, 9).permute(2, 1, 0).contiguous()            # [9][Cin][Cout]
    out, st = _stem_det(x, wp, b, Cout, stride, tag)
    gx, ppc = _stem_grid_x(H, W, Cout, stride), 256 // (Cout // 8)
    Ho, Wo = H // stride, W // stride
    nq = _cdiv(Ho * (Wo // 4), gx * ppc)         # pixel quads per thread
    if H == 288:
        assert gx == 148 * 8 and nq > 1, (gx, nq)
    ref = F.conv2d(x.double(), w.double(), b.double(), stride=stride, padding=1).permute(0, 2, 3, 1)
    mag = F.conv2d(x.double().abs(), w.double().abs(), b.double().abs(), stride=stride, padding=1).permute(0, 2, 3, 1)
    e32 = (9 * Cin + 1) * U * mag        # an fp32 fma chain from the bias over 9 Cin terms
    _report(tag, (out.double() - ref).abs(), 0.5 * _ulp_bf16(ref.abs() + e32) + e32 + 1e-300)
    # statistics of the stored values: a thread's 4 nq pixels, the ppc thread slots in order, the gx CTA slots (stat_parts_reduce)
    y = out.double().reshape(B, Ho * Wo, Cout)
    sref = torch.stack([y.sum(1), (y * y).sum(1)], 2)
    smag = torch.stack([y.abs().sum(1), (y * y).sum(1)], 2)
    nadd = 4 * nq + ppc + _cdiv(gx, 8) + 8 + 1
    _report(f"{tag} stats", (st.double() - sref).abs(), _sum_tol(nadd, smag))
    out_a = torch.empty_like(out)
    st_a = torch.zeros_like(st)
    fn = _L().pdae_stem_conv_bf16 if stride == 1 else _L().pdae_stem_conv_s2_bf16
    _native.check(fn(_p(x), _p(wp), _p(b), _p(out_a), _p(st_a), B, H, W, Cin, Cout, _stream()), "stem (default)")
    torch.cuda.synchronize()
    _assert_bitwise(f"{tag} out vs default", out, out_a)     # the same conv code: only the statistics flush differs
    _report(f"{tag} stats vs default", (st.double() - st_a.double()).abs(), _sum_tol(nadd + 4 * nq + ppc + gx + 1, smag))
    if B > 1 and H <= 32:
        _batch_invariance(tag, lambda i: (_stem_inputs(1, Cin, H, W, Cout, seed=70 + i)[0],),
                          lambda xb: _stem_det(xb[0], wp, b, Cout, stride, f"{tag} batch"))


def test_stem_det_rejects_a_shape_beyond_48k_of_shared_memory():
    B, Cin, H, W, Cout = 1, 4, 16, 16, 256          # (9 * 4 + 2 + 2 * 8) * 256 floats = 54 KiB
    x, w, b = _stem_inputs(B, Cin, H, W, Cout, seed=3)
    wp = w.reshape(Cout, Cin, 9).permute(2, 1, 0).contiguous()
    out = _nan((B, H, W, Cout), torch.bfloat16)
    st = _nan((B, Cout, 2))
    ws = _Workspace(_L().pdae_stem_conv_det_workspace_bytes(B, H, W, Cout, 1))
    rc = _L().pdae_stem_conv_bf16_det(_p(x), _p(wp), _p(b), _p(out), _p(st), B, H, W, Cin, Cout, 1, ws.ptr, ws.need, _stream())
    torch.cuda.synchronize()
    assert rc == PDAE_EINVAL and b"shared memory" in _L().pdae_last_error()
    assert torch.isnan(out.float()).all() and torch.isnan(st).all()
    ws.check_guard("stem_det 4->256")


# ---- conv_tc2: forward convolutions -----------------------------------------------------------------------------------
def _pow2_tile(n, cap):
    t = 1
    while t * 2 <= cap and n % (t * 2) == 0:
        t *= 2
    return t


def _tc2_tiles_per_image(H, W):
    tw = _pow2_tile(W, 128)
    th = _pow2_tile(H, 128 // tw)
    return (W // tw) * (H // th), 128 // (tw * th)


def _bf16(t):
    return t.to(torch.bfloat16)


class _Tc2Conv:
    """Inputs, weights and float64 reference of one conv_tc2 forward.  mode: conv (3x3, or 1x1 with k=1), skip (+ 1x1 conv of a
    second input), skip2 (+ 1x1 conv of a two-tensor concat), split (split-operand input [hi|lo|hi], weights [W_hi|W_hi|W_lo])
    or s2 (3x3 stride 2, H x W the input size)."""

    def __init__(self, mode, B, H, W, Cin, Cout, k, bn, out_bf16, res, seed, images=None):
        g = torch.Generator().manual_seed(seed)
        rnd = lambda *s: torch.randn(*s, generator=g)                            # noqa: E731
        self.mode, self.B, self.H, self.W, self.Cin, self.Cout, self.k, self.bn = mode, B, H, W, Cin, Cout, k, bn
        self.odt = torch.bfloat16 if out_bf16 else torch.float32
        self.Ho, self.Wo = (H // 2, W // 2) if mode == "s2" else (H, W)
        x = images if images is not None else rnd(B, H, W, Cin).to(DEV)
        self.x32 = x
        self.w = (rnd(Cout, Cin, k, k) / (k * Cin ** 0.5)).to(DEV)
        self.bias = (0.3 * rnd(Cout)).to(DEV)
        self.res = _bf16(rnd(B, H, W, Cout).to(DEV)).to(self.odt) if res else None
        if mode == "split":
            self.xin = _split3(x)
            wh = _bf16(self.w)
            wl = _bf16(self.w - wh.float())
            self.wp = torch.cat([wh, wh, wl], 1).reshape(Cout, 3 * Cin, k * k).permute(2, 0, 1).contiguous()
            self.xr, self.wr = x.double(), self.w.double()
        else:
            self.xin = _bf16(x).contiguous()
            self.wp = _bf16(self.w).reshape(Cout, Cin, k * k).permute(2, 0, 1).contiguous()
            self.xr, self.wr = self.xin.double(), _bf16(self.w).double()
        self.skips = []
        if mode in ("skip", "skip2"):
            cs = (192,) if mode == "skip" else (64, 128)
            self.w2 = _bf16((rnd(Cout, sum(cs)) / sum(cs) ** 0.5).to(DEV)).contiguous()
            self.skips = [_bf16(rnd(B, H, W, c).to(DEV)).contiguous() for c in cs]

    def create(self, out, stats):
        h = ctypes.c_void_p()
        L, odt = _L(), (PDAE_BF16 if self.odt == torch.bfloat16 else PDAE_F32)
        B, H, W, Cout = self.B, self.H, self.W, self.Cout
        Cop = self.xin.shape[3]
        if self.mode == "s2":
            rc = L.pdae_conv_tc2_create_s2_ex(ctypes.byref(h), _p(self.xin), _p(self.wp), _p(self.bias), _p(out), odt, _p(stats),
                                              B, H, W, Cop, Cout)
        elif self.mode == "skip":
            rc = L.pdae_conv_tc2_create_skip(ctypes.byref(h), _p(self.xin), _p(self.wp), _p(self.bias), _p(self.skips[0]),
                                             _p(self.w2), self.skips[0].shape[3], _p(out), odt, _p(stats), B, H, W, Cop, Cout,
                                             self.k, self.bn)
        elif self.mode == "skip2":
            a, b = self.skips
            rc = L.pdae_conv_tc2_create_skip2(ctypes.byref(h), _p(self.xin), _p(self.wp), _p(self.bias), _p(a), a.shape[3], _p(b),
                                              b.shape[3], _p(self.w2), _p(out), odt, _p(stats), B, H, W, Cop, Cout, self.k, self.bn)
        else:
            rc = L.pdae_conv_tc2_create(ctypes.byref(h), _p(self.xin), _p(self.wp), _p(self.bias), _p(self.res), _p(out), odt,
                                        _p(stats), B, H, W, Cop, Cout, self.k, 0, self.bn)
        _native.check(rc, f"conv_tc2 create ({self.mode})")
        return h

    def reference(self):
        """float64 output (NHWC) and the magnitude that bounds its fp32 evaluation, and the number of accumulated terms."""
        s = 2 if self.mode == "s2" else 1
        xr, wr = self.xr.permute(0, 3, 1, 2), self.wr
        y = F.conv2d(xr, wr, self.bias.double(), stride=s, padding=self.k // 2)
        mag = F.conv2d(xr.abs(), wr.abs(), self.bias.double().abs(), stride=s, padding=self.k // 2)
        nterm = self.k * self.k * self.xin.shape[3]
        if self.skips:
            xs = torch.cat(self.skips, 3).double().permute(0, 3, 1, 2)
            w2 = self.w2.double()[:, :, None, None]
            y, mag = y + F.conv2d(xs, w2), mag + F.conv2d(xs.abs(), w2.abs())
            nterm += xs.shape[1]
        if self.res is not None:
            r = self.res.double().permute(0, 3, 1, 2)
            y, mag = y + r, mag + r.abs()
        return _nhwc(y), _nhwc(mag), nterm

    def tol(self, ref, mag, nterm):
        e = (nterm + 3) * 2 * U * mag        # wgmma fp32 accumulation, then the bias and residual adds
        if self.mode == "split":             # a_hi w_hi + a_lo w_hi + a_hi w_lo misses at most 3.2 x 2^-18 |a w| per product
            e = e + 2.0 ** -16 * mag
        return (0.5 * _ulp_bf16(ref.abs() + e) + e if self.odt == torch.bfloat16 else e) + 1e-300

    def run_det(self, tag):
        out = torch.empty(self.B, self.Ho, self.Wo, self.Cout, dtype=self.odt, device=DEV)
        st = torch.empty(self.B, self.Cout, 2, device=DEV)
        h = self.create(out, st)
        try:
            need = _L().pdae_conv_tc2_det_workspace_bytes(h)
            P, _ = _tc2_tiles_per_image(self.Ho, self.Wo)
            assert need == (0 if P == 1 else self.B * P * self.Cout * 8), (need, P)
            return _det_run(tag, need, [out, st], lambda w, n: _L().pdae_conv_tc2_run(h, _stream()),
                            arm=lambda w, n: _L().pdae_conv_tc2_set_deterministic(h, w, n))
        finally:
            _L().pdae_conv_tc2_destroy(h)

    def run_default(self):
        out = _nan((self.B, self.Ho, self.Wo, self.Cout), self.odt)
        st = torch.zeros(self.B, self.Cout, 2, device=DEV)
        h = self.create(out, st)
        try:
            _native.check(_L().pdae_conv_tc2_run(h, _stream()), "conv_tc2 run (default)")
            torch.cuda.synchronize()
        finally:
            _L().pdae_conv_tc2_destroy(h)
        return out, st


def _check_stats(tag, out, st, st_default, P, HW):
    """DET statistics vs float64 sums of the stored values: a tile holds at most 128 of an image's pixels (any order: 128
    roundings), then stat_parts_reduce adds the P tile slots; the atomic twin adds at most HW values in some order."""
    y = out.double().reshape(out.shape[0], HW, -1)
    sref = torch.stack([y.sum(1), (y * y).sum(1)], 2)
    smag = torch.stack([y.abs().sum(1), (y * y).sum(1)], 2)
    nadd = 128 + _cdiv(P, 8) + 8 + 1
    _report(f"{tag} stats", (st.double() - sref).abs(), _sum_tol(nadd, smag))
    _report(f"{tag} stats vs default", (st.double() - st_default.double()).abs(), _sum_tol(nadd + HW + 1, smag))


TC2_CASES = [  # (mode, B, H, W, Cin, Cout, k, bn, out_bf16, res)
    ("conv", 2, 16, 8, 64, 64, 3, 0, False, True),      # one 16x8 tile per image: need 0, the slots are ch_stats itself
    ("conv", 2, 16, 8, 64, 128, 3, 0, True, False),
    ("conv", 2, 32, 32, 64, 128, 3, 64, False, True),   # eight tiles per image, BN 64
    ("conv", 2, 32, 16, 128, 256, 3, 256, True, False),  # BN 256
    ("conv", 3, 16, 16, 64, 128, 3, 128, True, True),   # BN 128, bf16 residual
    ("conv", 3, 8, 8, 64, 128, 3, 0, False, True),      # two images per tile, masked batch tail
    ("conv", 3, 4, 4, 128, 64, 3, 0, True, False),      # eight images per tile, three of them real
    ("conv", 2, 16, 16, 128, 64, 1, 0, False, False),   # 1x1
    ("skip", 3, 8, 8, 64, 128, 3, 0, False, False),     # fused 1x1 skip conv, two images per tile
    ("skip", 2, 32, 32, 64, 64, 3, 0, True, False),
    ("skip2", 2, 16, 16, 64, 64, 3, 0, True, False),    # skip conv over a two-tensor concat
    ("skip2", 3, 8, 8, 128, 128, 3, 0, False, False),
    ("split", 2, 16, 16, 64, 64, 3, 0, False, True),    # split-operand input, K = 3 Cin: fp32-grade
    ("split", 2, 32, 32, 64, 128, 3, 0, False, False),
    ("s2", 2, 32, 32, 64, 128, 3, 0, False, False),     # stride 2 with statistics, both output dtypes
    ("s2", 3, 16, 16, 64, 64, 3, 0, True, False),
]


def _tc2_id(c):
    mode, B, H, W, Cin, Cout, k, bn, ob, res = c
    return f"{mode}-b{B}-{H}x{W}-{Cin}-{Cout}-k{k}-bn{bn}" + ("-bf16" if ob else "-f32") + ("-res" if res else "")


@pytest.mark.parametrize("case", TC2_CASES, ids=[_tc2_id(c) for c in TC2_CASES])
def test_conv_tc2_det_matches_float64_and_the_default_kernel(case):
    mode, B, H, W, Cin, Cout, k, bn, out_bf16, res = case
    tag = f"conv_tc2 det {_tc2_id(case)}"
    cv = _Tc2Conv(mode, B, H, W, Cin, Cout, k, bn, out_bf16, res, seed=Cin + Cout + H)
    out, st = cv.run_det(tag)
    ref, mag, nterm = cv.reference()
    _report(tag, (out.double() - ref).abs(), cv.tol(ref, mag, nterm))
    out_d, st_d = cv.run_default()
    # The DET instantiation only changes the statistics epilogue; the k loop is the same code in the same order.
    _assert_bitwise(f"{tag} out vs default", out, out_d)
    P, _ = _tc2_tiles_per_image(cv.Ho, cv.Wo)
    _check_stats(tag, out, st, st_d, P, cv.Ho * cv.Wo)


@pytest.mark.parametrize("case", [("conv", 8, 8, 64, 128, False), ("conv", 4, 4, 128, 64, True), ("conv", 32, 32, 64, 64, False),
                                  ("skip", 8, 8, 64, 128, False), ("s2", 16, 16, 64, 64, True)],
                         ids=lambda c: f"{c[0]}-{c[1]}x{c[2]}")
def test_conv_tc2_det_is_batch_invariant(case):
    mode, H, W, Cin, Cout, ob = case
    g = torch.Generator().manual_seed(H + Cin)
    imgs = [torch.randn(1, H, W, Cin, generator=g).to(DEV) for _ in range(5)]

    def run(xb):
        cv = _Tc2Conv(mode, xb[0].shape[0], H, W, Cin, Cout, 3, 0, ob, False, seed=5, images=xb[0])
        if cv.skips:     # the skip input follows the image too
            cv.skips = [_bf16(xb[0][..., :1].expand(-1, -1, -1, 192) * 0.5).contiguous()]
        return cv.run_det(f"conv_tc2 det batch {mode} {H}x{W}")
    _batch_invariance(f"conv_tc2 det {mode} {H}x{W}", lambda i: (imgs[i],), run)


# ---- conv_tc2: split-K Linear -----------------------------------------------------------------------------------------
def _tc2_det_splitk(Cin, Cout):
    """tc2_det_splitk (conv_tc2.cu): (k ranges, k-blocks per range, k-blocks)."""
    BN = 128 if Cout % 128 == 0 else 64
    ntn = Cout // BN
    want = 1 if ntn >= 128 else 128 // ntn
    kb = Cin // 64
    kc = _cdiv(kb, want)
    return _cdiv(kb, kc), kc, kb


SPLITK_CASES = [  # (B, Cin, Cout, what)
    (1, 512, 1024, "even"),
    (5, 1344, 1024, "ragged"),      # 21 k-blocks in ranges of 2: the last range holds one
    (8, 2048, 512, "even"),
    (256, 512, 512, "even"),        # two 128-row tiles
    (5, 256, 8256, "single"),       # Cout / BN = 129 >= 128: a single k range
]


@pytest.mark.parametrize("B,Cin,Cout,what", SPLITK_CASES)
def test_conv_tc2_det_splitk_matches_float64_and_the_atomic_kernel(B, Cin, Cout, what):
    tag = f"conv_tc2 det split-K B={B} {Cin}->{Cout}"
    g = torch.Generator().manual_seed(B + Cin)
    x = _bf16(torch.randn(B, Cin, generator=g).to(DEV)).contiguous()
    w = _bf16((torch.randn(Cout, Cin, generator=g) / Cin ** 0.5).to(DEV)).contiguous()
    bias = (0.3 * torch.randn(Cout, generator=g)).to(DEV)
    splits, kc, kb = _tc2_det_splitk(Cin, Cout)
    assert {"single": splits == 1, "ragged": splits > 1 and kb % kc != 0, "even": splits > 1 and kb % kc == 0}[what], \
        (splits, kc, kb)
    out = torch.empty(B, Cout, device=DEV)
    h = ctypes.c_void_p()
    _native.check(_L().pdae_conv_tc2_create_splitk(ctypes.byref(h), _p(x), _p(w), _p(bias), _p(out), B, Cin, Cout), "splitk")
    try:
        need = _L().pdae_conv_tc2_det_workspace_bytes(h)
        assert need == splits * B * Cout * 4, (need, splits)
        # the repeat with no zeroing in between is the "out no longer needs zeroing" promise
        (got,) = _det_run(tag, need, [out], lambda w_, n: _L().pdae_conv_tc2_run(h, _stream()),
                          arm=lambda w_, n: _L().pdae_conv_tc2_set_deterministic(h, w_, n))
    finally:
        _L().pdae_conv_tc2_destroy(h)
    xd, wd = x.double(), w.double()
    ref = xd @ wd.t() + bias.double()
    mag = xd.abs() @ wd.abs().t() + bias.double().abs()
    # each range: a wgmma chain over its 64 kc products; then the ranges in order and the bias
    tol = (Cin + splits + 2) * 2 * U * mag + 1e-300
    _report(tag, (got.double() - ref).abs(), tol)
    out_a = torch.zeros(B, Cout, device=DEV)
    h = ctypes.c_void_p()
    _native.check(_L().pdae_conv_tc2_create_splitk(ctypes.byref(h), _p(x), _p(w), _p(bias), _p(out_a), B, Cin, Cout), "splitk")
    try:
        _native.check(_L().pdae_conv_tc2_run(h, _stream()), "splitk run")
        torch.cuda.synchronize()
    finally:
        _L().pdae_conv_tc2_destroy(h)
    # the atomic kernel splits by the SM count: at most kb ranges
    _report(f"{tag} vs atomic", (got.double() - out_a.double()).abs(), tol + (Cin + kb + 2) * 2 * U * mag)


# ---- conv_tc2: GEMM modes and the stride-2 data gradient (no statistics, no slots) --------------------------------------
def _plan_det_vs_default(tag, create, outs):
    """Run a plan made by create() once as it is and once switched to DET (need 0): the DET outputs must be bitwise those of
    the default kernel (the DET instantiations only compile out the unused statistics flush)."""
    h = create()
    try:
        for o in outs:
            _fill_nan(o)
        _native.check(_L().pdae_conv_tc2_run(h, _stream()), f"{tag} (default)")
        torch.cuda.synchronize()
        default = [o.clone() for o in outs]
        need = _L().pdae_conv_tc2_det_workspace_bytes(h)
        assert need == 0, need
        got = _det_run(tag, need, outs, lambda w, n: _L().pdae_conv_tc2_run(h, _stream()),
                       arm=lambda w, n: _L().pdae_conv_tc2_set_deterministic(h, w, n))
    finally:
        _L().pdae_conv_tc2_destroy(h)
    for i, (a, b) in enumerate(zip(got, default)):
        _assert_bitwise(f"{tag} output {i} vs default", a, b)
    return got


def _mm_ref(a, b, K, odt):
    """float64 a @ b^T over the last two dims and its tolerance (a wgmma chain of K terms; half a bf16 ulp for a bf16 store)."""
    ref = a.double() @ b.double().transpose(-1, -2)
    e = (K + 2) * 2 * U * (a.double().abs() @ b.double().abs().transpose(-1, -2))
    return ref, (0.5 * _ulp_bf16(ref.abs() + e) + e if odt == torch.bfloat16 else e) + 1e-300


@pytest.mark.parametrize("odt", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_gemm_tc2_det_is_the_default_kernel_and_matches_float64(odt):
    batch, M, N, K = 3, 256, 192, 128
    g = torch.Generator().manual_seed(31)
    a = _bf16(torch.randn(batch, M, K, generator=g).to(DEV)).contiguous()
    b = _bf16(torch.randn(batch, N, K, generator=g).to(DEV)).contiguous()
    out = torch.empty(batch, M, N, dtype=odt, device=DEV)
    od = PDAE_BF16 if odt == torch.bfloat16 else PDAE_F32

    def create():
        h = ctypes.c_void_p()
        _native.check(_L().pdae_gemm_tc2_create(ctypes.byref(h), _p(a), K, M * K, _p(b), K, N * K, _p(out), od, N, M * N, batch, M,
                                                N, K), "gemm_tc2_create")
        return h
    (got,) = _plan_det_vs_default(f"gemm_tc2 det {odt}", create, [out])
    ref, tol = _mm_ref(a, b, K, odt)
    _report(f"gemm_tc2 det {odt}", (got.double() - ref).abs(), tol)


@pytest.mark.parametrize("a_mn,b_mn", [(0, 1), (1, 0), (1, 1)])
def test_gemm_tc2_major_det_is_the_default_kernel_and_matches_float64(a_mn, b_mn):
    batch, M, N, K = 2, 128, 128, 192
    g = torch.Generator().manual_seed(37 + 2 * a_mn + b_mn)
    A = _bf16(torch.randn(batch, M, K, generator=g).to(DEV))
    Bm = _bf16(torch.randn(batch, N, K, generator=g).to(DEV))
    a_st = A.transpose(1, 2).contiguous() if a_mn else A.contiguous()        # [K][M] or [M][K]
    b_st = Bm.transpose(1, 2).contiguous() if b_mn else Bm.contiguous()
    out = torch.empty(batch, M, N, device=DEV)

    def create():
        h = ctypes.c_void_p()
        _native.check(_L().pdae_gemm_tc2_create_major(ctypes.byref(h), _p(a_st), a_mn, a_st.shape[2], a_st[0].numel(), _p(b_st),
                                                      b_mn, b_st.shape[2], b_st[0].numel(), _p(out), N, M * N, batch, M, N, K),
                      "gemm_tc2_create_major")
        return h
    (got,) = _plan_det_vs_default(f"gemm_tc2_major det a_mn={a_mn} b_mn={b_mn}", create, [out])
    ref, tol = _mm_ref(A, Bm, K, torch.float32)
    _report(f"gemm_tc2_major det a_mn={a_mn} b_mn={b_mn}", (got.double() - ref).abs(), tol)


def test_gemm_tc2_softmax_and_softmax_grad_det_are_the_default_kernels():
    """The softmax epilogues' accuracy against torch is test_gpu_conv_tc's; here their DET plans must be the same kernels."""
    batch, M, N, K, alpha = 2, 128, 128, 64, 0.125
    g = torch.Generator().manual_seed(41)
    q = _bf16(torch.randn(batch, M, K, generator=g).to(DEV)).contiguous()
    k = _bf16(torch.randn(batch, N, K, generator=g).to(DEV)).contiguous()
    P = torch.empty(batch, M, N, dtype=torch.bfloat16, device=DEV)

    def create_sm():
        h = ctypes.c_void_p()
        _native.check(_L().pdae_gemm_tc2_softmax_create(ctypes.byref(h), _p(q), K, M * K, _p(k), K, N * K, _p(P), N, M * N, batch,
                                                        M, N, K, alpha), "gemm_tc2_softmax_create")
        return h
    (p_det,) = _plan_det_vs_default("gemm_tc2_softmax det", create_sm, [P])
    P.copy_(p_det)
    dO = _bf16(torch.randn(batch, M, K, generator=g).to(DEV)).contiguous()
    v = _bf16(torch.randn(batch, N, K, generator=g).to(DEV)).contiguous()
    dS = torch.empty(batch, M, N, dtype=torch.bfloat16, device=DEV)

    def create_sg():
        h = ctypes.c_void_p()
        _native.check(_L().pdae_gemm_tc2_softmax_grad_create(ctypes.byref(h), _p(dO), K, M * K, _p(v), K, N * K, _p(P), N, M * N,
                                                             _p(dS), N, M * N, batch, M, N, K, alpha),
                      "gemm_tc2_softmax_grad_create")
        return h
    (ds,) = _plan_det_vs_default("gemm_tc2_softmax_grad det", create_sg, [dS])
    assert torch.isfinite(ds.float()).all()


def test_conv_tc2_s2_dgrad_det_is_the_default_kernel_and_matches_float64():
    B, H, W, Cin, Cout = 2, 16, 16, 64, 128
    g = torch.Generator().manual_seed(43)
    w = _bf16((torch.randn(Cout, Cin, 3, 3, generator=g) / (3 * Cout ** 0.5)).to(DEV))
    dy = _bf16(torch.randn(B, H // 2, W // 2, Cout, generator=g).to(DEV)).contiguous()
    wt = w.permute(2, 3, 1, 0).reshape(9, Cin, Cout).contiguous()       # wt[3 ky + kx][ci][co] = w[co][ci][ky][kx]
    dx = torch.empty(B, H, W, Cin, device=DEV)

    def create():
        h = ctypes.c_void_p()
        _native.check(_L().pdae_conv_tc2_create_s2_dgrad(ctypes.byref(h), _p(dy), _p(wt), _p(dx), B, H, W, Cin, Cout),
                      "create_s2_dgrad")
        return h
    (got,) = _plan_det_vs_default("conv_tc2_s2_dgrad det", create, [dx])
    x = torch.zeros(B, Cin, H, W, dtype=torch.float64, device=DEV, requires_grad=True)
    F.conv2d(x, w.double(), stride=2, padding=1).backward(dy.double().permute(0, 3, 1, 2))
    xa = torch.zeros_like(x, requires_grad=True)
    F.conv2d(xa, w.double().abs(), stride=2, padding=1).backward(dy.double().abs().permute(0, 3, 1, 2))
    tol = (9 * Cout + 2) * 2 * U * _nhwc(xa.grad) + 1e-300
    _report("conv_tc2_s2_dgrad det", (got.double() - _nhwc(x.grad)).abs(), tol)


# ---- conv_tc3 ---------------------------------------------------------------------------------------------------------
def _tc3_det_hook(tag, B, P, Cout, result):
    def hook(h, out, stats):
        need = _L().pdae_conv_tc3_det_workspace_bytes(h)
        assert need == (0 if P == 1 else B * P * Cout * 8), (need, P)
        result.extend(_det_run(tag, need, [out, stats], lambda w, n: _L().pdae_conv_tc3_run(h, _stream()),
                           arm=lambda w, n: _L().pdae_conv_tc3_set_deterministic(h, w, n)))
    return hook


TC3_CASES = [  # (B, H, W, C1, C2, Cout, res, skip, bn)
    (2, 16, 8, 64, 0, 64, False, False, 0),       # one 16x8 tile per image: need 0
    (3, 32, 32, 128, 0, 128, True, False, 0),     # 8 tiles per image, residual
    (2, 64, 64, 64, 64, 64, False, True, 0),      # 32 tiles per image, concat + fused skip
    (1, 48, 24, 64, 128, 128, False, True, 64),   # forced BN = 64
]


@pytest.mark.parametrize("x3", [False, True], ids=["bf16", "split"])
@pytest.mark.parametrize("case", TC3_CASES, ids=lambda c: "x".join(map(str, c[:6])))
def test_conv_tc3_det_matches_float64_and_the_default_kernel(case, x3):
    B, H, W, C1, C2, Cout, res, skip, bn = case
    P = (H // 16) * (W // 8)
    for out_bf16 in ((False,) if x3 else (True, False)):
        tag = f"conv_tc3 det {case} x3={x3} out_bf16={out_bf16}"
        got = []
        _tc3_run(B, H, W, C1, C2, Cout, x3, out_bf16, res, skip, bn, det=_tc3_det_hook(tag, B, P, Cout, got))
        out, st = got
        out_d, st_d, _ = _tc3_run(B, H, W, C1, C2, Cout, x3, out_bf16, res, skip, bn)
        # the DET instantiation only changes where the statistics go; the operand path and k loop are the same code
        _assert_bitwise(f"{tag} out vs default", out, out_d)
        _check_stats(tag, out, st, st_d, P, H * W)


@pytest.mark.parametrize("H,W,x3", [(16, 8, False), (32, 32, True)])
def test_conv_tc3_det_is_batch_invariant(H, W, x3):
    """_tc3_run draws every input from one seeded generator in the order (sources, ab, ...): image i of a batch is therefore
    not a fixed tensor, so the batches are built here and passed through a patched source."""
    C, Cout = 64, 64
    g = torch.Generator().manual_seed(H)
    imgs = [(torch.randn(1, H, W, C, generator=g) * 1.5 + 0.3).to(DEV) for _ in range(5)]
    abs_ = [torch.stack([1.0 + 0.3 * torch.randn(1, C, generator=g), 0.2 * torch.randn(1, C, generator=g)], 1).to(DEV)
            for _ in range(5)]
    w = (torch.randn(Cout, C, 3, 3, generator=g) / (3.0 * C ** 0.5)).to(DEV)
    bias = (0.1 * torch.randn(Cout, generator=g)).to(DEV)
    P = (H // 16) * (W // 8)

    def run(xb):
        x, ab = xb
        Bn = x.shape[0]
        sdt = torch.float32 if x3 else torch.bfloat16
        s1 = x.to(sdt).contiguous()
        if x3:
            hi = w.to(torch.bfloat16)
            wp = torch.stack([hi, (w - hi.float()).to(torch.bfloat16)], 0).reshape(2, Cout, C, 9).permute(3, 0, 1, 2).contiguous()
        else:
            wp = w.reshape(Cout, C, 9).permute(2, 0, 1).to(torch.bfloat16).contiguous()
        out = torch.empty(Bn, H, W, Cout, device=DEV)
        st = torch.empty(Bn, Cout, 2, device=DEV)
        h = ctypes.c_void_p()
        _native.check(_L().pdae_conv_tc3_create(ctypes.byref(h), _p(s1), C, None, 0, PDAE_F32 if x3 else PDAE_BF16,
                                                _p(ab.contiguous()), 1, _p(wp), _p(bias), None, 0, None, 0, None, None, _p(out),
                                                PDAE_F32, _p(st), Bn, H, W, Cout, 0), "conv_tc3_create")
        got = []
        try:
            _tc3_det_hook(f"conv_tc3 det batch {H}x{W}", Bn, P, Cout, got)(h, out, st)
        finally:
            _L().pdae_conv_tc3_destroy(h)
        return got
    _batch_invariance(f"conv_tc3 det {H}x{W} x3={x3}", lambda i: (imgs[i], abs_[i]), run)


# ---- wgrad_tc ---------------------------------------------------------------------------------------------------------
def _wg_det_splits(B, H, W, Cin, Cout, k, split, s2):
    """wg_det_splits (wgrad_tc.cu) on the plan's shape: (splits, k-tiles per split, k-tiles)."""
    if s2:
        H, W = H // 2, W // 2
    a_is_act = Cout % 128 != 0
    pair = a_is_act and Cin % 128 != 0
    Ma, Nb = (Cin, Cout) if a_is_act else (Cout, Cin)
    BN = 128 if Nb % 128 == 0 else 64
    mch = Ma // 64 if pair else Ma // 128
    taps = k * k
    tw = _pow2_tile(W, 64)
    th = _pow2_tile(H, 64 // tw)
    tn = 64 // (tw * th)
    kt = (W // tw) * (H // th) * _cdiv(B, tn)
    groups = ((taps + 1) // 2 if pair else taps) * mch * (Nb // BN)
    n = taps * Cin * Cout
    best, bk = 0.0, kt
    for s in range(1, kt + 1):
        kk = _cdiv(kt, s)
        if s > 1 and _cdiv(kt, kk) != s:
            continue
        cost = _cdiv(groups * s, 132) * kk + (s * n / 750000.0 * (1 if split else 3) if s > 1 else 0.0)
        if s == 1 or cost < best:
            best, bk = cost, kk
    return _cdiv(kt, bk), bk, kt


WGRAD_CASES = [  # (plan, B, H, W, Cin, Cout, k, what)
    ("split", 1, 8, 8, 128, 128, 3, "one"),        # one split: the kernel stores straight into dw
    ("split", 32, 16, 16, 256, 256, 3, "ragged"),  # 7 splits of 19 k-tiles over 128: the last holds 14
    ("split", 2, 32, 32, 64, 64, 3, "many"),       # pair mode
    ("bf16", 8, 32, 32, 128, 128, 3, "ragged"),    # 13 splits of 10 k-tiles over 128
    ("bf16", 1, 8, 8, 64, 128, 1, "one"),
    ("bf16_s2", 4, 32, 32, 128, 128, 3, "many"),
]


@pytest.mark.parametrize("plan,B,H,W,Cin,Cout,k,what", WGRAD_CASES)
def test_wgrad_tc_det_matches_float64_and_the_atomic_kernel(plan, B, H, W, Cin, Cout, k, what):
    tag = f"wgrad_tc det {plan} B={B} {H}x{W} {Cin}->{Cout} k={k}"
    s2 = plan == "bf16_s2"
    g = torch.Generator().manual_seed(B + H + Cin)
    Hd, Wd = (H // 2, W // 2) if s2 else (H, W)
    act = (torch.randn(B, H, W, Cin, generator=g) * 1.3 + 0.2).to(DEV)
    dy = (torch.randn(B, Hd, Wd, Cout, generator=g) * 0.05).to(DEV)
    if plan == "split":
        a_in, d_in = _split3(act), _split3(dy)
        ad, dd = act.double(), dy.double()
    else:
        a_in, d_in = _bf16(act).contiguous(), _bf16(dy).contiguous()
        ad, dd = a_in.double(), d_in.double()
    splits, kpt, kt = _wg_det_splits(B, H, W, Cin, Cout, k, plan == "split", s2)
    assert {"one": splits == 1, "many": splits > 1, "ragged": splits > 1 and kt % kpt != 0}[what], (splits, kpt, kt)

    def create(dw):
        h = ctypes.c_void_p()
        L = _L()
        if plan == "split":
            rc = L.pdae_wgrad_tc_create(ctypes.byref(h), _p(a_in), _p(d_in), _p(dw), B, H, W, Cin, Cout, k)
        elif plan == "bf16":
            rc = L.pdae_wgrad_tc_create_bf16(ctypes.byref(h), _p(a_in), _p(d_in), _p(dw), B, H, W, Cin, Cout, k)
        else:
            rc = L.pdae_wgrad_tc_create_bf16_s2(ctypes.byref(h), _p(a_in), _p(d_in), _p(dw), B, H, W, Cin, Cout)
        _native.check(rc, f"{tag} create")
        return h
    dw = torch.empty(k * k, Cin, Cout, device=DEV)
    h = create(dw)
    try:
        need = _L().pdae_wgrad_tc_det_workspace_bytes(h)
        assert need == (0 if splits == 1 else splits * k * k * Cin * Cout * 4), (need, splits)
        (got,) = _det_run(tag, need, [dw], lambda w, n: _L().pdae_wgrad_tc_run(h, _stream()),
                          arm=lambda w, n: _L().pdae_wgrad_tc_set_deterministic(h, w, n))
    finally:
        _L().pdae_wgrad_tc_destroy(h)
    st = 2 if s2 else 1
    ref = wgrad_ref(ad, dd, k, st)
    mag = wgrad_ref(ad.abs(), dd.abs(), k, st)
    per = 3 if plan == "split" else 1          # products per term
    # a split's wgmma chain over its kpt * 64 pixels (per products each), then the splits in order
    tol = (per * 64 * kpt + splits + 2) * 2 * U * mag + 1e-300
    if plan == "split":                        # split-operand products: at most 3.2 x 2^-18 |a dy| each
        tol = tol + 2.0 ** -16 * mag
    _report(f"{tag} (splits={splits}, k-tiles/split={kpt}, k-tiles={kt})", (got.double() - ref).abs(), tol)
    dw_a = torch.zeros_like(dw)
    h = create(dw_a)
    try:
        _native.check(_L().pdae_wgrad_tc_run(h, _stream()), f"{tag} (atomic)")
        torch.cuda.synchronize()
    finally:
        _L().pdae_wgrad_tc_destroy(h)
    _report(f"{tag} vs atomic", (got.double() - dw_a.double()).abs(), tol + (per * 64 * kt + kt + 2) * 2 * U * mag)


# ---- CUDA-core backward: wgrad_simt_det, dgrad_simt_det, colsum_det ------------------------------------------------------
def _wgrad_simt_det_chunk(P, MK, Cout):
    """wgrad_simt_args (backward_simt.cu): the DET pixel chunk and chunk count (132 x 4 CTAs aimed for)."""
    tiles = _cdiv(MK, 64) * _cdiv(Cout, 64)
    splits = max(min(_cdiv(132 * 4, tiles), _cdiv(P, 256)), 1)
    chunk = _cdiv(_cdiv(P, splits), 16) * 16
    return chunk, _cdiv(P, chunk)


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,stride,nchw,a_silu,what", [
    (2, 8, 8, 64, 64, 3, 1, 0, 0, "one"),       # one chunk: workspace 0, written straight into dw
    (1, 33, 31, 16, 8, 3, 1, 0, 1, "ragged"),   # 1023 pixels in 256-pixel chunks: the last holds 255
    (3, 33, 31, 32, 70, 3, 2, 1, 1, "ragged"),  # NCHW input with SiLU, stride 2: 816 pixels in chunks of 208
    (6, 1, 1, 128, 1100, 1, 1, 0, 1, "one"),    # the Linear bank (B, 1, 1, E -> total)
])
def test_wgrad_simt_det_matches_float64_and_the_atomic_kernel(B, H, W, Cin, Cout, k, stride, nchw, a_silu, what):
    tag = f"wgrad_simt_det B={B} {H}x{W} {Cin}->{Cout} k={k} s={stride} nchw={nchw} silu={a_silu}"
    g = torch.Generator().manual_seed(13 + H)
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    x = torch.randn(B, Cin, H, W, generator=g).to(DEV)
    dy = torch.randn(B, Ho, Wo, Cout, generator=g).to(DEV)
    xin = x.contiguous() if nchw else x.permute(0, 2, 3, 1).contiguous()
    P, MK = B * Ho * Wo, k * k * Cin
    chunk, chunks = _wgrad_simt_det_chunk(P, MK, Cout)
    assert {"one": chunks == 1, "many": chunks > 1, "ragged": chunks > 1 and P % chunk != 0}[what], (chunk, chunks)
    need = _L().pdae_conv2d_wgrad_simt_det_workspace_bytes(B, H, W, Cin, Cout, k, stride, pad)
    assert need == (0 if chunks == 1 else chunks * MK * Cout * 4), need
    dw = torch.empty(MK, Cout, device=DEV)
    (got,) = _det_run(tag, need, [dw], lambda w, n: _L().pdae_conv2d_wgrad_simt_det(
        _p(xin), nchw, a_silu, _p(dy), _p(dw), B, H, W, Cin, Cout, k, stride, pad, w, n, _stream()))
    a = F.silu(x.double()) if a_silu else x.double()
    dyn = dy.double().permute(0, 3, 1, 2)

    def wg(inp, grad):
        w_ = torch.nn.grad.conv2d_weight(inp, (Cout, Cin, k, k), grad, stride=stride, padding=pad)
        return w_.permute(2, 3, 1, 0).reshape(MK, Cout)
    ref, mag = wg(a, dyn), wg(a.abs(), dyn.abs())
    # a CTA's fp32 fma chain over its chunk, then the chunk slots in order; SiLU(x) within 4u
    tol = (chunk + chunks + 8) * U * mag + 1e-300
    _report(f"{tag} (P={P}, chunk={chunk}, chunks={chunks})", (got.double() - ref).abs(), tol)
    dw_a = torch.zeros_like(dw)
    _native.check(_L().pdae_conv2d_wgrad_simt(_p(xin), nchw, a_silu, _p(dy), _p(dw_a), B, H, W, Cin, Cout, k, stride, pad,
                                              _stream()), "wgrad_simt")
    torch.cuda.synchronize()
    # the atomic kernel: its own chunks (at most 256 pixels more per chain), one atomic per chunk
    _report(f"{tag} vs atomic", (got.double() - dw_a.double()).abs(), tol + (chunk + 256 + _cdiv(P, 16) + 8) * U * mag)


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,stride,acc,what", [
    (5, 1, 1, 96, 1024, 1, 1, 0, "wide"),       # wide Linear: 16 slots of 64 rows
    (33, 1, 1, 512, 1100, 1, 1, 0, "wide"),     # 18 slots, the last one 12 rows
    (4, 1, 1, 64, 1023, 1, 1, 0, "default"),    # Cout < 1024: the default path
    (3, 1, 1, 96, 1024, 1, 1, 1, "accumulate"),  # accumulate=1: the default path, which adds
    (2, 8, 8, 32, 48, 3, 2, 1, "accumulate"),
])
def test_dgrad_simt_det_matches_float64_and_the_default_kernel(B, H, W, Cin, Cout, k, stride, acc, what):
    tag = f"dgrad_simt_det B={B} {H}x{W} {Cin}<-{Cout} k={k} s={stride} acc={acc}"
    g = torch.Generator().manual_seed(5 + Cout)
    pad = k // 2
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (k * Cin ** 0.5)).to(DEV)
    dy = torch.randn(B, Ho, Wo, Cout, generator=g).to(DEV)
    wt = w.reshape(Cout, Cin, k * k).permute(2, 0, 1).contiguous()
    dx0 = torch.randn(B, H, W, Cin, generator=g).to(DEV)
    need = _L().pdae_conv2d_dgrad_simt_det_workspace_bytes(B, H, W, Cin, Cout, k, stride, pad, acc)
    assert need == (_cdiv(Cout, 64) * B * Cin * 4 if what == "wide" else 0), need
    dx = dx0.clone()
    (got,) = _det_run(tag, need, [dx], lambda w_, n: _L().pdae_conv2d_dgrad_simt_det(
        _p(dy), _p(wt), _p(dx), B, H, W, Cin, Cout, k, stride, pad, acc, w_, n, _stream()), prefill=not acc, repeat=not acc)
    x = torch.zeros(B, Cin, H, W, device=DEV, dtype=torch.float64, requires_grad=True)
    F.conv2d(x, w.double(), stride=stride, padding=pad).backward(dy.double().permute(0, 3, 1, 2))
    xa = torch.zeros_like(x, requires_grad=True)
    F.conv2d(xa, w.double().abs(), stride=stride, padding=pad).backward(dy.double().abs().permute(0, 3, 1, 2))
    ref, mag = _nhwc(x.grad), _nhwc(xa.grad)
    base = dx0.double() if acc else 0.0
    if acc:
        mag = mag + dx0.double().abs()
    # wide: each 64-row slot an fp32 chain, then the slots in order; default: one chain over k*k*Cout terms (+ the add)
    nadd = 64 + _cdiv(Cout, 64) + 2 if what == "wide" else k * k * Cout + 2
    _report(tag, (got.double() - base - ref).abs(), _sum_tol(nadd, mag))
    dx_a = dx0.clone()
    _native.check(_L().pdae_conv2d_dgrad_simt(_p(dy), _p(wt), _p(dx_a), B, H, W, Cin, Cout, k, stride, pad, acc, _stream()),
                  "dgrad_simt")
    torch.cuda.synchronize()
    if what == "wide":      # the atomic split-K kernel: 64-row chains added in any order
        _report(f"{tag} vs atomic", (got.double() - dx_a.double()).abs(), _sum_tol(2 * nadd, mag))
    else:                   # the DET entry point runs the default kernel itself
        _assert_bitwise(f"{tag} vs default", got, dx_a)


def _colsum_det_rows(M):
    rows = (M // 592 + 7) // 8 * 8
    return min(max(rows, 32), 512)


@pytest.mark.parametrize("M,N,offset,what", [
    (32, 128, 0, "one"),        # one chunk: written straight into out
    (37, 512, 0, "ragged"),     # two chunks of 32 rows, the second holds 5
    (70000, 256, 0, "many"),
    (513, 3, 0, "scalar"),      # N = 3: the scalar kernel
    (1000, 66, 0, "scalar"),    # N % 4 != 0
    (4096, 128, 1, "scalar"),   # dy one float past a 16-byte boundary: the scalar kernel
])
def test_colsum_det_matches_float64_and_the_atomic_kernel(M, N, offset, what):
    tag = f"colsum_det M={M} N={N} offset={offset}"
    g = torch.Generator().manual_seed(M + N)
    buf = torch.randn(M * N + offset, generator=g).to(DEV)
    dy = buf[offset:].view(M, N)
    rows = _colsum_det_rows(M)
    chunks = _cdiv(M, rows)
    assert what != "ragged" or (chunks > 1 and M % rows != 0), (rows, chunks)
    assert what != "one" or chunks == 1
    need = _L().pdae_colsum_det_workspace_bytes(M, N)
    assert need == (0 if chunks == 1 else chunks * N * 4), need
    out = torch.empty(N, device=DEV)
    (got,) = _det_run(tag, need, [out], lambda w, n: _L().pdae_colsum_det(ctypes.c_void_p(dy.data_ptr()), M, N, _p(out), w, n,
                                                                           _stream()))
    ref, mag = dy.double().sum(0), dy.double().abs().sum(0)
    nadd = rows + chunks + 8       # a chunk's rows (any tree inside the CTA), then the chunk slots in order
    _report(tag, (got.double() - ref).abs(), _sum_tol(nadd, mag))
    out_a = torch.zeros(N, device=DEV)
    _native.check(_L().pdae_colsum(ctypes.c_void_p(dy.data_ptr()), M, N, _p(out_a), _stream()), "colsum")
    torch.cuda.synchronize()
    _report(f"{tag} vs atomic", (got.double() - out_a.double()).abs(), _sum_tol(nadd + M + 1, mag))


# ---- GroupNorm backward ------------------------------------------------------------------------------------------------
def _gn_bwd_ppc(B, HW):
    ppc = 256
    while ppc > 8 and B * _cdiv(HW, ppc) < 592:
        ppc >>= 1
    return ppc


SUMS_CASES = [  # (C1, C2, B, H, W, rs, silu)
    (64, 0, 2, 8, 8, RESAMPLE_NONE, 1),
    (96, 0, 3, 18, 14, RESAMPLE_NONE, 0),
    (192, 0, 3, 16, 16, RESAMPLE_DOWN2, 1),
    (128, 0, 2, 16, 16, RESAMPLE_DOWN2, 0),
    (64, 32, 3, 8, 8, RESAMPLE_UP2, 1),
    (64, 64, 2, 8, 8, RESAMPLE_UP2, 0),
    (384, 512, 2, 16, 16, RESAMPLE_NONE, 1),     # concat
    (6144, 0, 2, 4, 4, RESAMPLE_NONE, 1),        # the channel limit
]


@pytest.mark.parametrize("C1,C2,B,H,W,rs,silu", SUMS_CASES)
def test_gn_bwd_sums_det_matches_float64_and_the_atomic_kernel(C1, C2, B, H, W, rs, silu):
    C, HW = C1 + C2, H * W
    tag = f"gn_bwd_sums_det C={C1}+{C2} B={B} {H}x{W} {RS_NAMES[rs]} silu={silu}"
    Ho, Wo = _out_hw(H, W, rs)
    x1, x2 = _inputs(B, H, W, C1, C2, seed=C + H)
    g = torch.Generator().manual_seed(C)
    ab = torch.stack([1.0 + 0.5 * torch.randn(B, C, generator=g), 0.5 * torch.randn(B, C, generator=g)], 1).to(DEV)
    dy = torch.randn(B, Ho, Wo, C, generator=g).to(DEV)
    need = _L().pdae_gn_bwd_sums_det_workspace_bytes(B, H, W, C)
    ppc = _gn_bwd_ppc(B, HW)
    P = _cdiv(HW, ppc)
    assert need == B * P * C * 8, need
    S = torch.empty(B, C, 2, device=DEV)
    (got,) = _det_run(tag, need, [S], lambda w, n: _L().pdae_gn_bwd_sums_det(
        _p(x1), C1, _p(x2), C2, _p(ab), _p(dy), silu, rs, B, H, W, _p(S), w, n, _stream()))
    x = _cat_nchw(x1, x2)
    a, b = ab[:, 0].double()[:, :, None, None], ab[:, 1].double()[:, :, None, None]
    u = a * x + b
    g_rt = _resample_t(dy.double().permute(0, 3, 1, 2), rs)
    g_abs = _resample_t(dy.double().abs().permute(0, 3, 1, 2), rs)
    gather = 3 * U * g_abs if rs == RESAMPLE_UP2 else 0.0          # the four-term fp32 sum of UP2
    if silu:
        sg = torch.sigmoid(u)
        dsl = sg * (1 + u * (1 - sg))
        du = g_rt * dsl
        # u = fma(a, x, b) (one rounding, |silu''| <= 0.5); dsilu with expf and three more roundings: 8u(1 + |u|)
        ddu = g_abs * (0.5 * U * u.abs() + 8 * U * (1 + u.abs())) + gather * dsl.abs() + U * du.abs()
    else:
        du, ddu = g_rt, gather + 0.0 * g_rt
    R = 256 // min(C // 4, 256)
    nb = _cdiv(ppc, R) + R + _cdiv(P, 8) + 8 + 1   # a thread's pixels, the CTA's rows in order, stat_parts_reduce
    ref = torch.stack([du.sum((2, 3)), (du * x).sum((2, 3))], 2)
    tol = torch.stack([nb * U * du.abs().sum((2, 3)) + ddu.sum((2, 3)),
                       (nb + 1) * U * (du * x).abs().sum((2, 3)) + (ddu * x.abs()).sum((2, 3))], 2) + 1e-300
    _report(tag, (got.double() - ref).abs(), tol)
    S_a = torch.zeros_like(S)
    _native.check(_L().pdae_gn_bwd_sums(_p(x1), C1, _p(x2), C2, _p(ab), _p(dy), silu, rs, B, H, W, _p(S_a), _stream()),
                  "gn_bwd_sums")
    torch.cuda.synchronize()
    nb_a = ppc + P + 2
    tol_a = torch.stack([nb_a * U * du.abs().sum((2, 3)), (nb_a + 1) * U * (du * x).abs().sum((2, 3))], 2)
    _report(f"{tag} vs atomic", (got.double() - S_a.double()).abs(), tol + tol_a)


COEF_CASES = [  # (B, C, HW, emb, dgamma, dbeta)
    (3, 64, 64, True, True, True),
    (2, 96, 252, False, True, True),
    (3, 512, 256, True, True, False),
    (2, 2048, 16, True, True, True),     # the channel limit: more channels than the 1024 threads
    (3, 256, 64, True, False, False),    # no dgamma / dbeta: no workspace (NULL)
]


@pytest.mark.parametrize("B,C,HW,use_emb,want_dg,want_db", COEF_CASES)
def test_gn_bwd_coef_det_matches_float64(B, C, HW, use_emb, want_dg, want_db):
    tag = f"gn_bwd_coef_det B={B} C={C} HW={HW} emb={int(use_emb)} dgamma={int(want_dg)} dbeta={int(want_db)}"
    g = torch.Generator().manual_seed(B * C + HW)
    cpg, n = C // 32, HW * (C // 32)
    # statistics of a plausible activation: group mean m, variance v, as the fp64 sums gn_stats leaves
    m = 0.5 * torch.randn(B, 32, generator=g, dtype=torch.float64)
    v = 0.5 + torch.rand(B, 32, generator=g, dtype=torch.float64)
    sums = torch.stack([m * n, (v + m * m) * n], 2).to(DEV)
    S = (torch.randn(B, C, 2, generator=g) * HW ** 0.5).to(DEV)
    gamma = (1.0 + 0.3 * torch.randn(C, generator=g)).to(DEV)
    beta = (0.3 * torch.randn(C, generator=g)).to(DEV)
    if use_emb:
        _, emb, eld = _bank(B, C, 5)
        _, embz, zld = _bank(B, C, 6)
        dbank_e, dbank_z = torch.empty(B, eld, device=DEV), torch.empty(B, zld, device=DEV)
        demb, dembz = dbank_e[:, 20:20 + 2 * C], dbank_z[:, 20:20 + 2 * C]
    else:
        emb = embz = demb = dembz = dbank_e = dbank_z = None
        eld = zld = 0
    kk = torch.empty(B, 3, C, device=DEV)
    dgamma = torch.empty(C, device=DEV) if want_dg else None
    dbeta = torch.empty(C, device=DEV) if want_db else None
    outs = [t for t in (kk, dgamma, dbeta, dbank_e, dbank_z) if t is not None]
    need = _L().pdae_gn_bwd_coef_det_workspace_bytes(B, C) if (want_dg or want_db) else 0
    assert need == 2 * B * C * 4 or not (want_dg or want_db)

    def run(w, nb):
        return _L().pdae_gn_bwd_coef_det(_p(S), _p(sums), _p(gamma), _p(beta), _p(emb), eld, _p(embz), zld, B, C, HW, EPS, _p(kk),
                                         _p(dgamma), _p(dbeta), _p(demb), eld, _p(dembz), zld, w if need else None, nb, _stream())
    got = _det_run(tag, need, outs, run)
    kk_g = got.pop(0)
    dg_g = got.pop(0) if want_dg else None
    db_g = got.pop(0) if want_db else None
    # float64 reference from the kernel's fp32 scale / gain values (s = 1 + e, zs = 1 + z, gt = gamma s zs, all fp32); every
    # other step is fp64 and the results are rounded to fp32 once (+ fp64 rounding noise, bounded by 2^-45 of the magnitudes)
    one = torch.ones(B, C, device=DEV)
    s = (1.0 + emb[:, :C]) if use_emb else one
    sh = emb[:, C:].double() if use_emb else 0.0 * one.double()
    zs = (1.0 + embz[:, :C]) if use_emb else one
    gt = (gamma[None] * s * zs).double()
    s, zs = s.double(), zs.double()
    sd = sums.double()
    mean = (sd[..., 0] / n).repeat_interleave(cpg, 1)
    var = (sd[..., 1] / n - (sd[..., 0] / n) ** 2).repeat_interleave(cpg, 1)
    rstd = 1.0 / torch.sqrt(var + EPS)
    S1, S2 = S[..., 0].double(), S[..., 1].double()
    dbt, dgt = S1, rstd * (S2 - mean * S1)
    m_dgt = rstd * (S2.abs() + (mean * S1).abs())
    grp = lambda t: t.reshape(B, 32, cpg).sum(2).repeat_interleave(cpg, 1)     # noqa: E731
    gA, gB = grp(gt * dbt), grp(gt * dgt)
    k0, k1 = rstd * gt, -rstd * rstd * gB / n
    k2 = -rstd * gA / n - k1 * mean
    m1 = rstd * rstd / n * grp(gt.abs() * m_dgt)
    m2 = rstd / n * grp((gt * dbt).abs()) + m1 * mean.abs()
    F64 = 2.0 ** -45
    ref = torch.stack([k0, k1, k2], 1)
    tol = U * ref.abs() + F64 * torch.stack([k0.abs(), m1, m2], 1) + 1e-300
    _report(f"{tag} kk", (kk_g.double() - ref).abs(), tol)
    for name, got_p, part, mpart in (("dgamma", dg_g, dgt * s * zs, m_dgt * (s * zs).abs()), ("dbeta", db_g, dbt * s * zs, None)):
        if got_p is None:
            continue
        mpart = part.abs() if mpart is None else mpart
        # per image one rounding to fp32 (the slot), then the B slots added in order
        t = (B + 1) * U * mpart.sum(0) + F64 * mpart.sum(0) + 1e-300
        _report(f"{tag} {name}", (got_p.double() - part.sum(0)).abs(), t)
    if use_emb:
        gd, bd = gamma.double()[None], beta.double()[None]
        e_ref = torch.cat([(dgt * gd + dbt * bd) * zs, dbt * zs], 1)
        e_mag = torch.cat([(m_dgt * gd.abs() + dbt.abs() * bd.abs()) * zs.abs(), (dbt * zs).abs()], 1)
        z_ref = torch.cat([dgt * gd * s + dbt * (bd * s + sh), dbt], 1)
        z_mag = torch.cat([m_dgt * (gd * s).abs() + dbt.abs() * ((bd * s).abs() + sh.abs()), dbt.abs()], 1)
        de, dz = got
        _report(f"{tag} demb", (de[:, 20:20 + 2 * C].double() - e_ref).abs(), U * e_ref.abs() + F64 * e_mag + 1e-300)
        # beta * s + sh is evaluated in fp32 (two roundings) before it meets dbt in fp64
        z_fp32 = torch.cat([2 * U * dbt.abs() * ((bd * s).abs() + sh.abs()), 0.0 * dbt], 1)
        _report(f"{tag} dembz", (dz[:, 20:20 + 2 * C].double() - z_ref).abs(), U * z_ref.abs() + z_fp32 + F64 * z_mag + 1e-300)
        for bank in (de, dz):     # nothing outside the (scale | shift) block is written
            assert torch.isnan(bank[:, :20]).all() and torch.isnan(bank[:, 20 + 2 * C:]).all(), f"{tag}: write outside demb"


# ---- embedding_bwd_det ------------------------------------------------------------------------------------------------
def test_embedding_bwd_det_matches_float64_and_the_atomic_kernel():
    g = torch.Generator().manual_seed(21)
    B, E, rows = 37, 130, 7
    idx = torch.tensor([i % 3 for i in range(B - 2)] + [4, 4], dtype=torch.int64).to(DEV)  # rows 3, 5, 6 unused; 6 > max index
    d = torch.randn(B, E, generator=g).to(DEV)
    dw = torch.empty(rows, E, device=DEV)
    (got,) = _det_run("embedding_bwd_det", 0, [dw], lambda w, n: _L().pdae_embedding_bwd_det(_p(d), _p(idx), _p(dw), B, E, rows,
                                                                                             _stream()))
    ref = torch.zeros(rows, E, dtype=torch.float64, device=DEV).index_add(0, idx, d.double())
    mag = torch.zeros(rows, E, dtype=torch.float64, device=DEV).index_add(0, idx, d.double().abs())
    cnt = torch.bincount(idx, minlength=rows).double()[:, None].to(DEV)
    for r in (3, 5, 6):
        assert bool((got[r] == 0).all()), f"embedding_bwd_det: unused row {r} is not 0"
    _report("embedding_bwd_det", (got.double() - ref).abs(), cnt * U * mag + 1e-300)
    dw_a = torch.zeros(rows, E, device=DEV)
    _native.check(_L().pdae_embedding_bwd(_p(d), _p(idx), _p(dw_a), B, E, _stream()), "embedding_bwd")
    torch.cuda.synchronize()
    _report("embedding_bwd_det vs atomic", (got.double() - dw_a.double()).abs(), 2 * cnt * U * mag + 1e-300)


# ---- per-image metrics ------------------------------------------------------------------------------------------------
def _ssim_ref(a, b):
    """float64 SSIM map (metric/utils.py:35-56 with the fp32 window) and a first-order bound of the kernel's fp32 evaluation:
    the five windowed sums are fp32 fma chains of 121 terms, then about a dozen fp32 operations."""
    from pdae_b200.metric.utils import _window
    C = a.shape[1]
    w = _window(a.device).double()[None, None].expand(C, 1, 11, 11)
    cv = lambda t: F.conv2d(t, w, padding=5, groups=C)                        # noqa: E731
    a, b = a.double(), b.double()
    mu1, mu2, s11, s22, s12 = cv(a), cv(b), cv(a * a), cv(b * b), cv(a * b)
    e_mu1, e_mu2 = 122 * U * cv(a.abs()), 122 * U * cv(b.abs())
    e11, e22, e12 = 123 * U * s11, 123 * U * s22, 123 * U * cv((a * b).abs())
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    A = 2 * mu1 * mu2 + c1
    Bv = 2 * (s12 - mu1 * mu2) + c2
    Cd = mu1 ** 2 + mu2 ** 2 + c1
    Dd = (s11 - mu1 ** 2) + (s22 - mu2 ** 2) + c2
    dmu12 = mu1.abs() * e_mu2 + mu2.abs() * e_mu1 + e_mu1 * e_mu2 + U * (mu1 * mu2).abs()
    eA = 2 * dmu12 + 2 * U * A.abs()
    eB = 2 * (e12 + dmu12) + 4 * U * (s12.abs() + (mu1 * mu2).abs()) + U * Bv.abs()
    eC = 2 * (mu1.abs() * e_mu1 + mu2.abs() * e_mu2) + e_mu1 ** 2 + e_mu2 ** 2 + 3 * U * Cd.abs()
    eD = e11 + e22 + 2 * (mu1.abs() * e_mu1 + mu2.abs() * e_mu2) + e_mu1 ** 2 + e_mu2 ** 2 \
        + 5 * U * (s11.abs() + s22.abs() + mu1 ** 2 + mu2 ** 2)
    num, den = A * Bv, Cd * Dd
    e_num = eA * Bv.abs() + A.abs() * eB + eA * eB
    e_den = eC * Dd.abs() + Cd.abs() * eD + eC * eD
    den_lo = (den.abs() - e_den).clamp_min(1e-300)
    err = (e_num + (num / den).abs() * e_den) / den_lo + 3 * U * (num / den).abs()
    return num / den, err


@pytest.mark.parametrize("B,C,H,W", [(3, 3, 37, 29), (2, 1, 64, 61), (4, 3, 20, 45), (2, 3, 256, 255)])
def test_mse_and_ssim_det_match_float64_and_the_default_kernels(B, C, H, W):
    from pdae_b200.metric import utils as mu
    g = torch.Generator().manual_seed(B * H + W)
    a = torch.rand(B, C, H, W, generator=g).to(DEV)
    b = (a.cpu() + 0.1 * torch.randn(B, C, H, W, generator=g)).to(DEV)
    n = C * H * W
    tag = f"B={B} C={C} {H}x{W}"
    L = _L()
    # mse: per block an fp64 sum of fp32 squared differences (two roundings each), the slots in order
    need = L.pdae_mse_det_workspace_bytes(B, n)
    nblk = min(_cdiv(n, 256 * 8), 64)
    assert need == B * nblk * 8 and n % (256 * 8 * nblk) != 0, (need, nblk)   # a ragged last block stride
    out = torch.empty(B, device=DEV)
    (mse,) = _det_run(f"mse_det {tag}", need, [out], lambda w, nb: L.pdae_mse_per_image_det(_p(a), _p(b), B, n, w, nb, _p(out),
                                                                                           _stream()))
    d2 = ((a.double() - b.double()) ** 2).reshape(B, -1)
    ref = d2.mean(1)
    tol = 3 * U * ref + (n + 8) * U53 * ref + 1e-300     # (a - b) and its square in fp32, fp64 sums, one rounding to fp32
    _report(f"mse_det {tag}", (mse.double() - ref).abs(), tol)
    ws = torch.empty(B, dtype=torch.float64, device=DEV)
    out_a = torch.empty(B, device=DEV)
    _native.check(L.pdae_mse_per_image(_p(a), _p(b), B, n, _p(ws), _p(out_a), _stream()), "mse_per_image")
    torch.cuda.synchronize()
    _report(f"mse_det vs default {tag}", (mse.double() - out_a.double()).abs(), 2 * tol)
    # ssim: per 16x16 tile an fp64 sum of fp32 per-pixel values, the tiles in order
    need = L.pdae_ssim_det_workspace_bytes(B, C, H, W)
    assert need == B * C * _cdiv(H, 16) * _cdiv(W, 16) * 8, need
    win = mu._window(a.device)
    out = torch.empty(B, device=DEV)
    (ssim,) = _det_run(f"ssim_det {tag}", need, [out], lambda w, nb: L.pdae_ssim_per_image_det(
        _p(a), _p(b), _p(win), B, C, H, W, w, nb, _p(out), _stream()))
    smap, serr = _ssim_ref(a, b)
    ref = smap.reshape(B, -1).mean(1)
    tol = serr.reshape(B, -1).mean(1) + U * ref.abs() + (n + 8) * U53 * smap.abs().reshape(B, -1).mean(1) + 1e-300
    _report(f"ssim_det {tag}", (ssim.double() - ref).abs(), tol)
    ws = torch.empty(B, dtype=torch.float64, device=DEV)
    _native.check(L.pdae_ssim_per_image(_p(a), _p(b), _p(win), B, C, H, W, _p(ws), _p(out_a), _stream()), "ssim_per_image")
    torch.cuda.synchronize()
    # the same per-pixel values: only the fp64 order of the sum and the final rounding differ
    t2 = 2 * (U * ref.abs() + (n + 8) * U53 * smap.abs().reshape(B, -1).mean(1)) + 1e-300
    _report(f"ssim_det vs default {tag}", (ssim.double() - out_a.double()).abs(), t2)
    # the metric functions take the DET kernels under torch.use_deterministic_algorithms
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        assert torch.equal(_bits(mu.calculate_mse(a, b)), _bits(mse))
        assert torch.equal(_bits(mu.calculate_ssim(a, b)), _bits(ssim))
    finally:
        torch.use_deterministic_algorithms(prev)

    def run(xb):
        x, y = xb
        Bn = x.shape[0]
        o1, o2 = torch.empty(Bn, device=DEV), torch.empty(Bn, device=DEV)
        w1 = _Workspace(L.pdae_mse_det_workspace_bytes(Bn, n))
        w2 = _Workspace(L.pdae_ssim_det_workspace_bytes(Bn, C, H, W))
        _native.check(L.pdae_mse_per_image_det(_p(x), _p(y), Bn, n, w1.ptr, w1.need, _p(o1), _stream()), "mse_det")
        _native.check(L.pdae_ssim_per_image_det(_p(x), _p(y), _p(win), Bn, C, H, W, w2.ptr, w2.need, _p(o2), _stream()), "ssim_det")
        torch.cuda.synchronize()
        return [o1, o2]
    _batch_invariance(f"mse/ssim det {tag}", lambda i: (a[i % B:i % B + 1] * (1 + 0.1 * i), b[i % B:i % B + 1]), run)
