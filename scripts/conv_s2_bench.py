"""Micro-benchmark of the stride-2 bf16 tensor-core convs (conv_tc2 forward and data gradient, wgrad_tc weight gradient) vs
their fp32 CUDA-core counterparts (conv2d_simt, conv2d_dgrad_simt, conv2d_wgrad_simt) on the semantic encoders' 3x3
stride-2 shapes.  TFLOP/s are algorithmic: 2 * B * (H/2) * (W/2) * Cin * Cout * 9 per contraction.
usage: python scripts/conv_s2_bench.py [--batch 32]"""
import argparse
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from pdae_b200 import _native

SHAPES = [(32, 64, 128), (16, 128, 128), (8, 128, 128),                        # 64-px encoder: (input H = W, Cin, Cout)
          (64, 64, 128), (32, 128, 256), (16, 256, 256), (8, 256, 256)]        # 128-px encoders
DEV = "cuda"
p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None


def timeit(fn, n=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3     # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    B = ap.parse_args().batch
    L = _native.lib()
    props = torch.cuda.get_device_properties(0)
    print(f"{props.name}, batch {B}; us per call and algorithmic TFLOP/s", flush=True)
    for H, Cin, Cout in SHAPES:
        W, Ho, Wo = H, H // 2, H // 2
        x = torch.randn(B, H, W, Cin, device=DEV)
        w = torch.randn(Cout, Cin, 3, 3, device=DEV) / (3 * Cin ** 0.5)
        bias = torch.randn(Cout, device=DEV)
        dy = torch.randn(B, Ho, Wo, Cout, device=DEV) * 0.05
        xb, dyb, wb = x.to(torch.bfloat16), dy.to(torch.bfloat16), w.to(torch.bfloat16)
        w_f = w.reshape(Cout, Cin, 9).permute(2, 1, 0).contiguous()           # simt forward:  [tap][Cin][Cout] fp32
        w_tco = w.reshape(Cout, Cin, 9).permute(2, 0, 1).contiguous()         # simt dgrad:    [tap][Cout][Cin] fp32
        w_fb = wb.reshape(Cout, Cin, 9).permute(2, 0, 1).contiguous()         # tc forward:    [tap][Cout][Cin] bf16
        w_db = wb.reshape(Cout, Cin, 9).permute(2, 1, 0).contiguous()         # tc dgrad:      [tap][Cin][Cout] bf16
        out, out2 = torch.empty(B, Ho, Wo, Cout, device=DEV), torch.empty(B, Ho, Wo, Cout, device=DEV)
        dx, dx2 = torch.empty(B, H, W, Cin, device=DEV), torch.empty(B, H, W, Cin, device=DEV)
        dw, dw2 = torch.zeros(9, Cin, Cout, device=DEV), torch.zeros(9, Cin, Cout, device=DEV)
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        hf, hd, hw = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
        _native.check(L.pdae_conv_tc2_create_s2(ctypes.byref(hf), p(xb), p(w_fb), p(bias), p(out), B, H, W, Cin, Cout), "fwd")
        _native.check(L.pdae_conv_tc2_create_s2_dgrad(ctypes.byref(hd), p(dyb), p(w_db), p(dx), B, H, W, Cin, Cout), "dgrad")
        _native.check(L.pdae_wgrad_tc_create_bf16_s2(ctypes.byref(hw), p(xb), p(dyb), p(dw), B, H, W, Cin, Cout), "wgrad")
        runs = [
            ("forward", lambda: L.pdae_conv_tc2_run(hf, st),
             lambda: L.pdae_conv2d_simt(p(x), 0, 0, p(w_f), p(bias), None, p(out2), 0, B, H, W, Cin, Cout, 3, 2, 1, 0, st)),
            ("dgrad", lambda: L.pdae_conv_tc2_run(hd, st),
             lambda: L.pdae_conv2d_dgrad_simt(p(dy), p(w_tco), p(dx2), B, H, W, Cin, Cout, 3, 2, 1, 0, st)),
            ("wgrad", lambda: L.pdae_wgrad_tc_run(hw, st),
             lambda: L.pdae_conv2d_wgrad_simt(p(x), 0, 0, p(dy), p(dw2), B, H, W, Cin, Cout, 3, 2, 1, st)),
        ]
        fl = 2.0 * B * Ho * Wo * Cin * Cout * 9
        line = [f"{H:3d}x{W:<3d} {Cin:3d}->{Cout:3d}:"]
        for name, tc, simt in runs:
            t_tc, t_simt = timeit(tc), timeit(simt, 5)
            line.append(f"{name} {t_tc:7.1f} us {fl / t_tc / 1e6:6.1f} TF | simt {t_simt:8.1f} us {fl / t_simt / 1e6:5.1f} TF")
        # agreement with the fp32 CUDA-core results (bf16 operand rounding only)
        dw.zero_(); dw2.zero_()
        for _, tc, simt in runs:
            tc(); simt()
        torch.cuda.synchronize()
        rel = [float((a - b).norm() / b.norm()) for a, b in ((out, out2), (dx, dx2), (dw, dw2))]
        print("  ".join(line) + f"  rel-L2 vs simt {rel[0]:.1e} / {rel[1]:.1e} / {rel[2]:.1e}", flush=True)
        L.pdae_conv_tc2_destroy(hf)
        L.pdae_conv_tc2_destroy(hd)
        L.pdae_wgrad_tc_destroy(hw)


if __name__ == "__main__":
    main()
