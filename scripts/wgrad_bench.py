"""Micro-benchmark of wgrad_tc (split-operand and single-pass bf16) vs conv2d_wgrad_simt on the celeba64-proxy training shapes
(B=32).  usage: python scripts/wgrad_bench.py"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from pdae_b200 import _native

DEV = "cuda"
L = _native.lib()
p = lambda t: ctypes.c_void_p(t.data_ptr())


def split3(x):
    hi = x.to(torch.bfloat16)
    return torch.cat([hi, (x - hi.float()).to(torch.bfloat16), hi], -1).contiguous()


def timeit(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


st = None
for (B, H, W, Cin, Cout, k) in [(32, 32, 32, 128, 128, 3), (32, 32, 32, 256, 128, 3), (32, 16, 16, 256, 256, 3), (32, 16, 16, 512, 256, 3),
                                (32, 8, 8, 512, 512, 3), (32, 8, 8, 1024, 512, 3), (32, 64, 64, 128, 64, 3), (32, 64, 64, 64, 64, 3), (32, 64, 64, 192, 64, 3), (32, 16, 16, 256, 256, 1)]:
    act = torch.randn(B, H, W, Cin, device=DEV)
    dy = torch.randn(B, H, W, Cout, device=DEV) * 0.05
    dw = torch.zeros(k * k, Cin, Cout, device=DEV)
    dw2 = torch.zeros_like(dw)
    a3, d3 = split3(act), split3(dy)
    ab, db = act.to(torch.bfloat16), dy.to(torch.bfloat16)
    dwb = torch.zeros_like(dw)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    h, hb = ctypes.c_void_p(), ctypes.c_void_p()
    _native.check(L.pdae_wgrad_tc_create(ctypes.byref(h), p(a3), p(d3), p(dw), B, H, W, Cin, Cout, k), "create")
    _native.check(L.pdae_wgrad_tc_create_bf16(ctypes.byref(hb), p(ab), p(db), p(dwb), B, H, W, Cin, Cout, k), "create_bf16")
    t_tc = timeit(lambda: _native.check(L.pdae_wgrad_tc_run(h, st), "run"))
    t_bf = timeit(lambda: _native.check(L.pdae_wgrad_tc_run(hb, st), "run bf16"))
    t_simt = timeit(lambda: _native.check(L.pdae_conv2d_wgrad_simt(p(act), 0, 0, p(dy), p(dw2), B, H, W, Cin, Cout, k, 1, k // 2, st), "simt"), 3)
    dw.zero_(); dw2.zero_(); dwb.zero_()
    L.pdae_wgrad_tc_run(h, st); L.pdae_wgrad_tc_run(hb, st)
    L.pdae_conv2d_wgrad_simt(p(act), 0, 0, p(dy), p(dw2), B, H, W, Cin, Cout, k, 1, k // 2, st)
    torch.cuda.synchronize()
    rel = ((dw - dw2).abs().max() / dw2.abs().max()).item()
    rel_b = ((dwb - dw2).abs().max() / dw2.abs().max()).item()
    fl = 2.0 * B * H * W * Cin * Cout * k * k
    print(f"B{B} {H}x{W} {Cin}->{Cout} k{k}: wgrad_tc {t_tc:8.1f} us ({fl / t_tc / 1e6:7.1f} TF alg, {3 * fl / t_tc / 1e6:7.1f} exec)   "
          f"bf16 {t_bf:8.1f} us ({fl / t_bf / 1e6:7.1f} TF)   simt {t_simt:8.1f} us   rel diff {rel:.2e} (bf16 {rel_b:.2e})", flush=True)
    L.pdae_wgrad_tc_destroy(h)
    L.pdae_wgrad_tc_destroy(hb)
