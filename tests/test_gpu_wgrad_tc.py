"""wgrad_tc (tensor-core weight gradient of a stride-1 "same" conv, split-operand fp32-grade) through the C-ABI vs the float64
autograd weight gradient of F.conv2d on the device: both operand placements (dY or the activation on the M side), the tap-pair mode, both N tiles,
1x1 and 3x3, ragged batch tiles, split-K over many CTAs and a single-item CTA range."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from pdae_b200 import _native

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _split3(x):
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return torch.cat([hi, lo, hi], -1).contiguous()


def run_wgrad(B, H, W, Cin, Cout, k, seed=0):
    g = torch.Generator(device="cpu").manual_seed(77 + seed)
    act = (torch.randn(B, H, W, Cin, generator=g) * 1.3 + 0.2).to(DEV)
    dy = (torch.randn(B, H, W, Cout, generator=g) * 0.05).to(DEV)
    dw = torch.zeros(k * k, Cin, Cout, device=DEV)
    L = _native.lib()
    assert L.pdae_wgrad_tc_supported(H, W, Cin, Cout, k)
    a3, d3 = _split3(act), _split3(dy)
    h = ctypes.c_void_p()
    _native.check(L.pdae_wgrad_tc_create(ctypes.byref(h), _p(a3), _p(d3), _p(dw), B, H, W, Cin, Cout, k), "pdae_wgrad_tc_create")
    try:
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _native.check(L.pdae_wgrad_tc_run(h, st), "pdae_wgrad_tc_run")
        torch.cuda.synchronize()
    finally:
        L.pdae_wgrad_tc_destroy(h)
    return dw.double(), wgrad_ref(act.double(), dy.double(), k)


def wgrad_ref(act, dy, k, stride=1):
    """float64 autograd weight gradient of F.conv2d (padding k // 2) in the kernels' layout [tap][cin][cout]; act, dy NHWC."""
    Cin, Cout = act.shape[3], dy.shape[3]
    x = act.permute(0, 3, 1, 2)
    w = torch.zeros(Cout, Cin, k, k, device=act.device, dtype=act.dtype, requires_grad=True)
    F.conv2d(x, w, stride=stride, padding=k // 2).backward(dy.permute(0, 3, 1, 2))
    return w.grad.reshape(Cout, Cin, k * k).permute(2, 1, 0)


CASES = [
    (4, 16, 16, 128, 128, 3),     # dY on the M side, N tile 128
    (3, 8, 8, 256, 128, 3),       # two N chunks
    (2, 32, 32, 128, 64, 3),      # activation on the M side (Cout = 64), N tile 64
    (2, 32, 32, 64, 128, 3),      # dY on the M side, N tile 64
    (4, 16, 16, 128, 256, 1),     # 1x1, two M chunks
    (5, 4, 4, 128, 128, 3),       # 4x4 images: 4 images per box, ragged batch tile
    (1, 8, 8, 128, 128, 3),       # one k-tile per (tap, chunk) group: every CTA drains after a single item
    (32, 16, 16, 256, 256, 3),    # long split-K ranges
    (2, 32, 32, 64, 64, 3),       # neither side fills 128 rows: two taps of 64 channels share the accumulator (pair mode)
    (2, 16, 16, 192, 64, 3),      # pair mode, three M chunks
    (3, 16, 16, 64, 64, 1),       # pair mode with a single tap
]


@pytest.mark.parametrize("B,H,W,Cin,Cout,k", CASES)
def test_wgrad_tc_matches_float64_autograd(B, H, W, Cin, Cout, k):
    got, ref = run_wgrad(B, H, W, Cin, Cout, k)
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    # split-operand products carry ~2^-17 relative error per term, fp32 accumulation over B*H*W pixels
    assert err <= 2e-5 * scale + 1e-7, (err, scale)
