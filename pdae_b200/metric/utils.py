"""On-device evaluation metrics and wire formats (SURVEY.md §8(f) rows 3 and 4).

Mirrors the names of the reference's metric/utils.py (`calculate_mse` :62-63, `calculate_ssim` :56-60) so that
metric/mse/mse_metric.py:11 and metric/ssim/ssim_metric.py:11 can import from here unchanged, plus the two image
conversions every trainer/sampler spells inline:
  * `images.mul(0.5).add(0.5).mul(255).add(0.5).clamp(0,255).permute(0,2,3,1).to('cpu', torch.uint8)`
    (trainer/train_representation_learning.py:173-174) -> `images_to_uint8` (device uint8 NHWC, bit-exact);
  * torchvision `ToTensor()` + `Normalize(0.5, 0.5)` (dataset/ffhq.py:27-31) -> `uint8_to_images`.
Each is ONE kernel launch through the C-ABI; CUDA tensors only (no CPU fallback).
"""
from __future__ import annotations

import ctypes
import math

import torch

from .. import _native


def _stream(dev) -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _req(*ts: torch.Tensor) -> None:
    for t in ts:
        if not t.is_cuda:
            raise _native.NativeError("pdae_b200.metric: CUDA tensors required (no CPU fallback)")


def images_to_uint8(images: torch.Tensor) -> torch.Tensor:
    """fp32 NCHW in [-1,1] -> uint8 NHWC on the same device."""
    _req(images)
    x = images.float().contiguous()
    B, C, H, W = x.shape
    out = torch.empty((B, H, W, C), dtype=torch.uint8, device=x.device)
    _native.check(_native.lib().pdae_images_to_u8_nhwc(x.data_ptr(), out.data_ptr(), B, C, H, W, _stream(x.device)),
                  "pdae_images_to_u8_nhwc")
    return out


def uint8_to_images(u8: torch.Tensor) -> torch.Tensor:
    """uint8 NHWC -> normalised fp32 NCHW ((x/255 - 0.5)/0.5) on the same device."""
    _req(u8)
    if u8.dtype != torch.uint8 or u8.dim() != 4:
        raise ValueError("uint8_to_images: expected a uint8 [B,H,W,C] tensor")
    u8 = u8.contiguous()
    B, H, W, C = u8.shape
    out = torch.empty((B, C, H, W), dtype=torch.float32, device=u8.device)
    _native.check(_native.lib().pdae_u8_nhwc_to_images(u8.data_ptr(), out.data_ptr(), B, C, H, W, _stream(u8.device)),
                  "pdae_u8_nhwc_to_images")
    return out


def calculate_mse(img1: torch.Tensor, img2: torch.Tensor) -> torch.Tensor:
    """Per-image mean squared error over (C,H,W) (metric/utils.py:62-63)."""
    _req(img1, img2)
    if img1.shape != img2.shape:
        raise ValueError("calculate_mse: shape mismatch")
    a, b = img1.float().contiguous(), img2.float().contiguous()
    B = a.shape[0]
    out = torch.empty(B, dtype=torch.float32, device=a.device)
    L = _native.lib()
    if torch.are_deterministic_algorithms_enabled():   # per-block slots added in a fixed order: bitwise-reproducible
        nb = L.pdae_mse_det_workspace_bytes(B, a[0].numel())
        _native.check(min(int(nb), 0), "pdae_mse_det_workspace_bytes")
        ws = torch.empty(max(int(nb), 8), dtype=torch.uint8, device=a.device)
        _native.check(L.pdae_mse_per_image_det(a.data_ptr(), b.data_ptr(), B, a[0].numel(), ws.data_ptr(), ws.numel(),
                                               out.data_ptr(), _stream(a.device)), "pdae_mse_per_image_det")
        return out
    ws = torch.empty(B, dtype=torch.float64, device=a.device)
    _native.check(_native.lib().pdae_mse_per_image(a.data_ptr(), b.data_ptr(), B, a[0].numel(), ws.data_ptr(), out.data_ptr(),
                                                   _stream(a.device)), "pdae_mse_per_image")
    return out


_WINDOWS = {}


def _window(dev) -> torch.Tensor:
    """metric/utils.py:25-33: normalised fp32 1-D Gaussian (11 taps, sigma 1.5), outer product."""
    w = _WINDOWS.get(dev)
    if w is None:
        g = torch.tensor([math.exp(-(x - 5) ** 2 / float(2 * 1.5 ** 2)) for x in range(11)], dtype=torch.float32)
        g = (g / g.sum()).unsqueeze(1)
        w = _WINDOWS[dev] = g.mm(g.t()).float().contiguous().to(dev)
    return w


def calculate_ssim(img1: torch.Tensor, img2: torch.Tensor, window_size: int = 11) -> torch.Tensor:
    """Per-image SSIM (metric/utils.py:35-60); only the reference's window_size=11 is built."""
    _req(img1, img2)
    if window_size != 11:
        raise ValueError("calculate_ssim: window_size must be 11 (the only value the reference uses)")
    if img1.shape != img2.shape or img1.dim() != 4:
        raise ValueError("calculate_ssim: expected two [B,C,H,W] tensors of the same shape")
    a, b = img1.float().contiguous(), img2.float().contiguous()
    B, C, H, W = a.shape
    out = torch.empty(B, dtype=torch.float32, device=a.device)
    L = _native.lib()
    if torch.are_deterministic_algorithms_enabled():   # per-block slots added in a fixed order: bitwise-reproducible
        nb = L.pdae_ssim_det_workspace_bytes(B, C, H, W)
        _native.check(min(int(nb), 0), "pdae_ssim_det_workspace_bytes")
        ws = torch.empty(max(int(nb), 8), dtype=torch.uint8, device=a.device)
        _native.check(L.pdae_ssim_per_image_det(a.data_ptr(), b.data_ptr(), _window(a.device).data_ptr(), B, C, H, W,
                                                ws.data_ptr(), ws.numel(), out.data_ptr(), _stream(a.device)),
                      "pdae_ssim_per_image_det")
        return out
    ws = torch.empty(B, dtype=torch.float64, device=a.device)
    _native.check(_native.lib().pdae_ssim_per_image(a.data_ptr(), b.data_ptr(), _window(a.device).data_ptr(), B, C, H, W,
                                                    ws.data_ptr(), out.data_ptr(), _stream(a.device)), "pdae_ssim_per_image")
    return out
