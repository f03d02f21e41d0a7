"""Training path: forward plans that keep their intermediates + hand-written backward plans, exposed through
``torch.autograd.Function`` so the reference trainers' ``loss.backward()`` / DDP hooks / Adam / EMA code keeps working
(trainer/train_representation_learning.py:86-112).

Scope (the PDAE training step, diffusion/gaussian_diffusion.py:234-255): the semantic encoder (all parameters) and the
trainable half of the ShiftUNet (``label_emb``, ``shift_middle_block``, ``shift_output_blocks``, ``shift_out``); the frozen
half builds no graph in the reference either (its parameters and x_t do not require grad) -- it runs as a tensor-core plan
in the split-operand (fp32-grade) mode with the fused-prologue convs.  The trainable half keeps its fp32 activations for the
backward; its forward convs, the data gradients and the weight gradients of the stride-1 convs run on the tensor cores on
split operands (``Plan.train_tc``, ``bwd_plan``, ``pdae_wgrad_tc_*``).  GroupNorm / attention backward, the encoder and the
stride-2 / 3-channel convs stay fp32 on CUDA cores (``pdae_gn_bwd_*``, ``pdae_gemm_batched_simt``, ``pdae_softmax_bwd``,
``pdae_conv2d_wgrad_simt`` / ``pdae_conv2d_dgrad_simt``).  Gradients reach autograd through one ``pdae_unpack_grads`` launch
(``GradSink``).  Dropout is inverted dropout with masks drawn by torch's CUDA generator.

Mixed precision: a ShiftUNet / UNet training forward called inside ``torch.autocast("cuda")`` (the reference trainers'
``enable_amp``; either autocast dtype) builds separate bf16 trainers: the frozen half runs as a plain "bf16" plan, and the
forward convs, data gradients and weight gradients of the trainable convs are single-pass bf16 MMAs with fp32 accumulation.
An eligible attention block (T % 128 == 0, T <= 256, head width % 64 == 0) also runs its attention core on the tensor
cores: bf16 qkv and probabilities in the forward; in the backward the softmax gradient sits in the epilogue of the dO V^T
GEMM (``pdae_gemm_tc2_softmax_grad_create``) and dV / dQ / dK are GEMMs with MN-major operands
(``pdae_gemm_tc2_create_major``) written in fp32 into the qkv gradient.  Other activations, GroupNorm and every gradient stay
fp32, so the reference's ``GradScaler`` works unchanged.  The semantic encoder does the same: under autocast its stride-2 convs (forward, data and weight gradient through parity views,
``pdae_conv_tc2_create_s2*``, ``pdae_wgrad_tc_create_bf16_s2``) and its attention 1x1 convs are single-pass bf16 MMAs; its
3-channel stem and final Linear stay fp32 on CUDA cores.  The latent MLPSkipNet's training step under autocast runs every
Linear but time_embed as a bf16 MMA (split-K where the batch leaves SMs idle), its layers' linear_emb as one bank GEMM, and
writes each layer's bf16 GEMM operand from the fused modulate / LayerNorm / SiLU / dropout kernel (MLPTrainer._init_amp);
an MLPSkipNet whose widths are not multiples of 64 keeps the fp32 trainer.  Every forward-only call (sampling,
``infer_latents``, a frozen encoder, MLPSkipNet sampling) ignores autocast.
"""
from __future__ import annotations

import ctypes
import math
import warnings
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import _native
from .engine import Buf, BufView, Plan, RESAMPLE_NONE, _STREAM
from .model.module import AttentionBlock, Src

F32 = ctypes.c_float


_UNPACK_ITEM = np.dtype([("src", "<u8"), ("dst_off", "<i8"), ("shape", "<i4", (4,)), ("stride", "<i8", (4,)), ("add", "<i4"),
                         ("pad", "<i4")])       # = pdae_unpack_item (include/pdae_b200.h)
_UNPACK_CHUNK = 4096


class GradSink:
    """parameter -> (zero-initialised accumulation view in the backward plan, un-packing function).

    `collect()` hands every gradient to autograd in the parameter's own layout.  The un-packing functions are pure VIEWS of the
    backward plan's accumulator arena (permute / slice / transpose), so their (shape, strides, offset) are recorded once and
    one `pdae_unpack_grads` launch gathers all of them into a fresh flat buffer; the returned gradients are views of that
    buffer (autograd adopts them as `.grad` without a copy)."""

    def __init__(self):
        self.items: List[Tuple[torch.Tensor, BufView, Callable[[torch.Tensor], torch.Tensor], int]] = []
        self._launches = None     # [(items table, block map, n_blocks)] per contribution rank
        self._slots: Dict[int, Tuple[torch.Tensor, int, int]] = {}
        self._total = 0

    def add(self, param: torch.Tensor, view: BufView, nelems: int, unpack: Callable[[torch.Tensor], torch.Tensor]) -> None:
        self.items.append((param, view, unpack, nelems))

    def _build(self) -> None:
        rank: Dict[int, int] = {}
        rows: Dict[int, list] = {}
        dev = None
        for param, view, unpack, n in self.items:
            arena = view.buf.tensor
            dev = arena.device
            v = unpack(arena[view.off: view.off + n])
            if v.untyped_storage().data_ptr() != arena.untyped_storage().data_ptr() or v.numel() != param.numel() or v.dim() > 4:
                raise _native.NativeError("pdae_b200: a gradient un-packing function must be a <=4-D view of the accumulator")
            if id(param) not in self._slots:
                self._slots[id(param)] = (param, self._total, param.numel())
                self._total += (param.numel() + 3) // 4 * 4          # 16-byte aligned slots
            r = rank[id(param)] = rank.get(id(param), -1) + 1
            shape = [1] * (4 - v.dim()) + list(v.shape)
            stride = [0] * (4 - v.dim()) + list(v.stride())
            rows.setdefault(r, []).append((v.data_ptr(), self._slots[id(param)][1], shape, stride, 1 if r else 0, 0))
        self._launches = []
        for r in sorted(rows):
            tab = np.array([tuple(x) for x in rows[r]], dtype=_UNPACK_ITEM)
            pairs = [(i, c) for i, x in enumerate(rows[r])
                     for c in range((int(np.prod(x[2])) + _UNPACK_CHUNK - 1) // _UNPACK_CHUNK)]
            t_dev = torch.from_numpy(tab.view(np.uint8).reshape(-1)).to(dev)
            b_dev = torch.tensor(pairs, dtype=torch.int32, device=dev).contiguous()
            self._launches.append((t_dev, b_dev, len(pairs)))
        self._dev = dev

    def collect(self) -> Dict[int, torch.Tensor]:
        if not self.items:
            return {}
        if self._launches is None:
            self._build()
        # a fresh buffer per backward (the caching allocator makes this free): gradients handed out earlier stay valid for as
        # long as the caller holds them, exactly like autograd's own
        flat = torch.empty(self._total, dtype=torch.float32, device=self._dev)
        L = _native.lib()
        st = ctypes.c_void_p(torch.cuda.current_stream(self._dev).cuda_stream)
        for t_dev, b_dev, nb in self._launches:
            _native.check(L.pdae_unpack_grads(t_dev.data_ptr(), b_dev.data_ptr(), nb, _UNPACK_CHUNK, flat.data_ptr(), st),
                          "pdae_unpack_grads")
        return {pid: flat[off: off + n].view(p.shape) for pid, (p, off, n) in self._slots.items()}


def draw_dropout_masks(plan: Plan) -> None:
    """One Bernoulli(1-p) mask per active Dropout, drawn with torch's CUDA generator (the reference's Philox stream is not
    reproduced; parity tests feed the same masks to the oracle)."""
    for _, mask, p in plan.dropout_masks:
        mask.tensor.bernoulli_(1.0 - p)


def bwd_plan(dev, amp: bool = False, det: bool = False) -> Plan:
    """Backward plans are tensor-core plans: the data gradient of every eligible stride-1 conv runs on `conv_tc2` and its
    weight gradient on `wgrad_tc`, both in the fp32-grade split-operand "bf16x3" mode, or with `amp` in the single-pass
    "bf16" mode (Backward.conv); everything else in them is fp32 CUDA-core arithmetic.  `det`: the deterministic plan
    (torch.use_deterministic_algorithms): DET tensor-core kernels and the *_det CUDA-core reductions, no float atomics."""
    return Plan(dev, "bf16" if amp else "bf16x3", deterministic=det)


def autocast_active() -> bool:
    """Is the caller inside an enabled CUDA autocast region?  Either autocast dtype selects the bf16 training plans: there
    are no fp16 kernels, and bf16 has fp32's exponent range, so a GradScaler's scale never overflows them."""
    return torch.is_autocast_enabled("cuda")


class Backward:
    """Emission helpers for the backward plan (fp32 activations / gradients; eligible convs on the tensor cores)."""

    def __init__(self, BP: Plan, sink: GradSink):
        self.P = BP
        self.sink = sink
        self._fixed: Dict[int, Buf] = {}

    def fx(self, b):
        if b is None:
            return None
        if isinstance(b, BufView):
            return BufView(self.fx(b.buf), b.off)
        if b.fixed:
            return b
        k = id(b)
        if k not in self._fixed:
            self._fixed[k] = self.P.fixed(b.tensor)
        return self._fixed[k]

    # ---- CUDA-core reductions: the atomic kernels, or in a deterministic plan their *_det forms (slots summed in order) --
    def wgrad_simt(self, x, in_nchw: int, a_silu: int, dy, dw, B, H, W, Cin, Cout, k, stride, pad) -> None:
        P = self.P
        if not P.det:
            P.call("conv2d_wgrad_simt", x, in_nchw, a_silu, dy, dw, B, H, W, Cin, Cout, k, stride, pad, _STREAM)
            return
        n = P.L.pdae_conv2d_wgrad_simt_det_workspace_bytes(B, H, W, Cin, Cout, k, stride, pad)
        ws = P.det_workspace(n, "pdae_conv2d_wgrad_simt_det_workspace_bytes")
        P.call("conv2d_wgrad_simt_det", x, in_nchw, a_silu, dy, dw, B, H, W, Cin, Cout, k, stride, pad, ws,
               ctypes.c_int64(ws.nbytes), _STREAM, launches=2 if n else 1)

    def dgrad_simt(self, dy, wt, dx, B, H, W, Cin, Cout, k, stride, pad) -> None:
        P = self.P
        if not P.det:
            P.call("conv2d_dgrad_simt", dy, wt, dx, B, H, W, Cin, Cout, k, stride, pad, 0, _STREAM)
            return
        n = P.L.pdae_conv2d_dgrad_simt_det_workspace_bytes(B, H, W, Cin, Cout, k, stride, pad, 0)
        ws = P.det_workspace(n, "pdae_conv2d_dgrad_simt_det_workspace_bytes")
        P.call("conv2d_dgrad_simt_det", dy, wt, dx, B, H, W, Cin, Cout, k, stride, pad, 0, ws, ctypes.c_int64(ws.nbytes), _STREAM,
               launches=2 if n else 1)

    def colsum(self, dy, M: int, N: int, out) -> None:
        P = self.P
        if not P.det:
            P.call("colsum", dy, ctypes.c_int64(M), N, out, _STREAM)
            return
        n = P.L.pdae_colsum_det_workspace_bytes(M, N)
        ws = P.det_workspace(n, "pdae_colsum_det_workspace_bytes")
        P.call("colsum_det", dy, ctypes.c_int64(M), N, out, ws, ctypes.c_int64(ws.nbytes), _STREAM, launches=2 if n else 1)

    # ---- conv / linear ------------------------------------------------------------------------------------------
    def conv(self, x, dy: Buf, weight: torch.Tensor, bias: Optional[torch.Tensor], *, B, H, W, Cin, Cout, k, stride=1, pad=None,
             need_dx=True, in_nchw=False, a_silu=False, trainable=True, w_unpack=None) -> Optional[Buf]:
        """x: forward input of the conv (NHWC fp32, or NCHW if in_nchw); dy: grad of its output [B,Ho,Wo,Cout]."""
        P = self.P
        pad = k // 2 if pad is None else pad
        Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        kk = k * k
        same = stride == 1 and k in (1, 3) and pad == k // 2 and not in_nchw
        # 3x3 stride-2 conv in the "bf16" backward (the semantic encoder under autocast): data and weight gradient on the
        # tensor cores through parity views (conv_tc2.cu, wgrad_tc.cu), fed by one bf16 copy of dy
        s2 = (P.precision == "bf16" and stride == 2 and k == 3 and pad == 1 and not (in_nchw or a_silu)
              and bool(P.L.pdae_conv_s2_tc_supported(H, W, Cin, Cout)))
        # tensor-core operands: split [hi | lo | hi] blocks in the "bf16x3" backward, plain bf16 in the "bf16" (autocast) one
        ce = 3 if P.x3 else 1
        dy3 = None
        if trainable:
            dw = P.new_grad(kk * Cin * Cout)
            if s2:
                act = getattr(x, "tc_copy", None)     # left by the bf16 training forward (Plan.conv)
                if act is not None and tuple(act.shape) == (B, H, W, Cin):
                    act = self.fx(act)
                else:
                    act, _ = P.gn_apply(self.fx(x), Cin, None, 0, None, silu=False, resample=RESAMPLE_NONE, B=B, H=H, W=W,
                                        act_dtype=torch.bfloat16)
                dy3, _ = P.gn_apply(dy, Cout, None, 0, None, silu=False, resample=RESAMPLE_NONE, B=B, H=Ho, W=Wo,
                                    act_dtype=torch.bfloat16)
                P.call("wgrad_tc_bf16_s2", act, dy3, dw, B, H, W, Cin, Cout, flops=2.0 * B * Ho * Wo * Cin * Cout * kk)
            elif same and not a_silu and P.L.pdae_wgrad_tc_supported(H, W, Cin, Cout, k):
                # weight gradient on the tensor cores (wgrad_tc.cu): fp32-grade split products, or single-pass bf16
                a3 = getattr(x, "tc_copy", None)       # left by the tensor-core training forward (Plan.conv, train_tc)
                if a3 is not None and tuple(a3.shape) == (B, H, W, ce * Cin):
                    a3 = self.fx(a3)
                else:
                    a3, _ = P.gn_apply(self.fx(x), Cin, None, 0, None, silu=False, resample=RESAMPLE_NONE, B=B, H=H, W=W,
                                       act_dtype=torch.bfloat16)
                dy3, _ = P.gn_apply(dy, Cout, None, 0, None, silu=False, resample=RESAMPLE_NONE, B=B, H=H, W=W,
                                    act_dtype=torch.bfloat16)
                P.call("wgrad_tc" if P.x3 else "wgrad_tc_bf16", a3, dy3, dw, B, H, W, Cin, Cout, k,
                       flops=2.0 * B * H * W * Cin * Cout * kk)
            else:
                self.wgrad_simt(self.fx(x), int(in_nchw), int(a_silu), dy, dw, B, H, W, Cin, Cout, k, stride, pad)
            unpack = w_unpack or (lambda t, kk=kk, Cin=Cin, Cout=Cout: t.view(kk, Cin, Cout).permute(2, 1, 0))
            self.sink.add(weight, dw, kk * Cin * Cout, unpack)
            if bias is not None:
                db = P.new_grad(Cout)
                self.colsum(dy, B * Ho * Wo, Cout, db)
                self.sink.add(bias, db, Cout, lambda t: t)
        if not need_dx:
            return None
        if s2:
            # sub-pixel phases of dx, each a stride-1 correlation of dy with 1, 2, 2 or 4 taps of the transposed weights
            if dy3 is None:
                dy3, _ = P.gn_apply(dy, Cout, None, 0, None, silu=False, resample=RESAMPLE_NONE, B=B, H=Ho, W=Wo,
                                    act_dtype=torch.bfloat16)
            wt = P.pack((id(weight), "tc_s2_dgrad"), [weight],
                        lambda: weight.detach().reshape(Cout, Cin, kk).permute(2, 1, 0).to(torch.bfloat16))
            dx = P.new((B, H, W, Cin), torch.float32, "dx")
            P.call("conv_tc2_s2_dgrad", dy3, wt, dx, B, H, W, Cin, Cout, flops=2.0 * B * Ho * Wo * Cin * Cout * kk)
            return dx
        if same and P.use_tc(Cout, Cin, k, 1, H, W):
            # dgrad of a stride-1 "same" conv = conv of dy with the transposed, spatially flipped weights: on the tensor
            # cores in the split-operand (fp32-grade) mode -- dy is split [hi | lo | hi], W' packed [W'_hi | W'_hi | W'_lo] --
            # or, in the "bf16" backward, as one bf16 product of plain dy and W' ("tc" pack)
            if dy3 is None:
                dy3, _ = P.gn_apply(dy, Cout, None, 0, None, silu=False, resample=RESAMPLE_NONE, B=B, H=H, W=W,
                                    act_dtype=torch.bfloat16)
            dx = P.new((B, H, W, Cin), torch.float32, "dx")
            P.conv(dy3, weight, None, dx, B=B, H=H, W=W, Cin=Cout, Cout=Cin, k=k, wkey=(id(weight), "dgrad"),
                   w_transform=lambda w, Cout=Cout, Cin=Cin, k=k: w.reshape(Cout, Cin, k, k).flip(2, 3).transpose(0, 1).contiguous())
            return dx
        wt = P.pack((id(weight), "tco"), [weight], lambda: weight.detach().reshape(Cout, Cin, kk).permute(2, 0, 1).float())
        dx = P.new((B, H, W, Cin), torch.float32, "dx")
        self.dgrad_simt(dy, wt, dx, B, H, W, Cin, Cout, k, stride, pad)
        return dx

    # ---- GroupNorm (+AdaGN) + SiLU (+resample) --------------------------------------------------------------------
    def gn(self, src: Src, ab: Buf, sums: Buf, gn_mod: nn.GroupNorm, dy: Buf, *, silu: bool, resample: int, emb=None, embz=None,
           demb=None, dembz=None, add: Optional[Buf] = None, add_ld: int = 0, trainable=True, want_dx2=False):
        """dy: grad of the (resampled) normalised activation, all C channels.  Returns dx for the first C1 channels
        (and, with want_dx2, also the gradient of the second / skip source)."""
        P = self.P
        B, H, W, C1, C2 = src.B, src.H, src.W, src.C1, src.C2
        C = C1 + C2
        S = P.new((B, C, 2), torch.float32, "gn_bwd_S")
        if P.det:
            ws = P.det_workspace(P.L.pdae_gn_bwd_sums_det_workspace_bytes(B, H, W, C), "pdae_gn_bwd_sums_det_workspace_bytes")
            P.call("gn_bwd_sums_det", self.fx(src.b1), C1, self.fx(src.b2), C2, self.fx(ab), dy, int(silu), resample, B, H, W, S,
                   ws, ctypes.c_int64(ws.nbytes), _STREAM, launches=2)
        else:
            P.call("gn_bwd_sums", self.fx(src.b1), C1, self.fx(src.b2), C2, self.fx(ab), dy, int(silu), resample, B, H, W, S,
                   _STREAM)
        kk = P.new((B, 3, C), torch.float32, "gn_bwd_k")
        dg = db = None
        if trainable:
            dg, db = P.new_grad(C), P.new_grad(C)
            self.sink.add(gn_mod.weight, dg, C, lambda t: t)
            self.sink.add(gn_mod.bias, db, C, lambda t: t)
        e, eld = (self.fx(emb[0]).at(emb[1]), emb[2]) if emb is not None else (None, 0)
        z, zld = (self.fx(embz[0]).at(embz[1]), embz[2]) if embz is not None else (None, 0)
        de, deld = (demb[0].at(demb[1]), demb[2]) if demb is not None else (None, 0)
        dz, dzld = (dembz[0].at(dembz[1]), dembz[2]) if dembz is not None else (None, 0)
        coef = (S, self.fx(sums), P.param(gn_mod.weight), P.param(gn_mod.bias), e, eld, z, zld, B, C, H * W, F32(1e-5), kk, dg, db,
                de, deld, dz, dzld)
        if P.det:
            ws = P.det_workspace(P.L.pdae_gn_bwd_coef_det_workspace_bytes(B, C), "pdae_gn_bwd_coef_det_workspace_bytes")
            P.call("gn_bwd_coef_det", *coef, ws, ctypes.c_int64(ws.nbytes), _STREAM, launches=2 if trainable else 1)
        else:
            P.call("gn_bwd_coef", *coef, _STREAM)
        dx = P.new((B, H, W, C1), torch.float32, "gn_dx")
        dx2 = P.new((B, H, W, C2), torch.float32, "gn_dx_skip") if (want_dx2 and C2) else None
        P.call("gn_bwd_apply", self.fx(src.b1), C1, self.fx(src.b2), C2, self.fx(ab), kk, dy, int(silu), resample, B, H, W, add,
               add_ld, dx, dx2, _STREAM)
        return (dx, dx2) if want_dx2 else dx

    # ---- blocks ----------------------------------------------------------------------------------------------------
    def resblock(self, blk, sv: dict, d_out: Buf, demb, dembz, want_dx2=False):
        P = self.P
        x: Src = sv["x"]
        B, H, W, C = x.B, x.H, x.W, x.C
        Co, H2, W2, rs = blk.out_channels, sv["H2"], sv["W2"], sv["rs"]
        conv1, conv2, gn1, gn2 = blk.in_layers[2], blk.out_layers[3], blk.in_layers[0], blk.out_layers[0]
        d_act2 = self.conv(sv["act2"], d_out, conv2.weight, conv2.bias, B=B, H=H2, W=W2, Cin=Co, Cout=Co, k=3)
        if sv.get("mask") is not None:   # dropout backward: the same mask and 1/(1-p) scale
            P.call("mul_mask", d_act2, self.fx(sv["mask"]), F32(1.0 / (1.0 - blk.dropout)), ctypes.c_int64(B * H2 * W2 * Co), _STREAM)
        hsrc = Src(sv["h"], Co, B, H2, W2)
        d_h = self.gn(hsrc, sv["ab2"], sv["sums2"], gn2, d_act2, silu=True, resample=RESAMPLE_NONE, emb=sv["emb"], embz=sv["embz"],
                      demb=demb, dembz=dembz)
        d_act1 = self.conv(sv["act1"], d_h, conv1.weight, conv1.bias, B=B, H=H2, W=W2, Cin=C, Cout=Co, k=3)
        if sv["ident"]:
            add, add_ld = d_out, Co          # skip = x_upd(x): gathered through the same resample^T inside gn_bwd_apply
        else:
            sk = blk.skip_connection
            sk_in = sv["raw"] if sv["raw"] is not None else x.b1
            add = self.conv(sk_in, d_out, sk.weight, sk.bias, B=B, H=H2, W=W2, Cin=C, Cout=Co, k=sk.kernel_size[0])
            add_ld = C
        return self.gn(x, sv["ab1"], sv["sums1"], gn1, d_act1, silu=True, resample=rs, add=add, add_ld=add_ld,
                       want_dx2=want_dx2)

    def attention(self, blk: AttentionBlock, sv: dict, d_out: Buf) -> Buf:
        P = self.P
        x: Src = sv["x"]
        B, H, W, C = x.B, x.H, x.W, x.C
        T, heads = H * W, blk.num_heads
        ch = C // heads
        legacy = sv["legacy"]
        d_att = self.conv(sv["att"], d_out, blk.proj_out.weight, blk.proj_out.bias, B=B, H=H, W=W, Cin=C, Cout=C, k=1)
        qkv, probs = self.fx(sv["qkv"]), self.fx(sv["probs"])
        row = 3 * C
        hs = 3 * ch if legacy else ch
        ko, vo = (ch, 2 * ch) if legacy else (C, 2 * C)
        d_qkv = P.new((B, T, 3 * C), torch.float32, "d_qkv")
        alpha = 1.0 / math.sqrt(ch)
        TT = T * T
        if sv.get("tc") and P.precision == "bf16":
            # bf16 tensor-core attention backward (the forward kept bf16 qkv and probabilities): dO in bf16 once, then per head
            #   dS = alpha P (dO V^T - rowsum(P dO V^T))   (softmax gradient in the GEMM epilogue, bf16)
            #   dV = P^T dO,  dQ = dS K,  dK = dS^T Q      (MN-major operands, fp32 straight into d_qkv)
            d_o, _ = P.gn_apply(d_att, C, None, 0, None, silu=False, resample=RESAMPLE_NONE, B=B, H=H, W=W,
                                act_dtype=torch.bfloat16)
            dS = P.new((B * heads, T, T), torch.bfloat16, "att_dS")
            for h in range(heads):
                q, k, v, o = h * hs, h * hs + ko, h * hs + vo, h * ch
                P.gemm_tc(d_o.at(o), C, T * C, qkv.at(v), row, T * row, dS.at(h * TT), T, heads * TT, batch=B, M=T, N=T, K=ch,
                          out_dtype=torch.bfloat16, softmax_grad=(probs.at(h * TT), T, heads * TT, alpha))
                P.gemm_tc(probs.at(h * TT), T, heads * TT, d_o.at(o), C, T * C, d_qkv.at(v), row, T * row, batch=B, M=T, N=ch,
                          K=T, out_dtype=torch.float32, a_mn=True, b_mn=True)
                P.gemm_tc(dS.at(h * TT), T, heads * TT, qkv.at(k), row, T * row, d_qkv.at(q), row, T * row, batch=B, M=T, N=ch,
                          K=T, out_dtype=torch.float32, b_mn=True)
                P.gemm_tc(dS.at(h * TT), T, heads * TT, qkv.at(q), row, T * row, d_qkv.at(k), row, T * row, batch=B, M=T, N=ch,
                          K=T, out_dtype=torch.float32, a_mn=True, b_mn=True)
            d_xn = self.conv(sv["xn"], d_qkv, blk.qkv.weight, blk.qkv.bias, B=B, H=H, W=W, Cin=C, Cout=3 * C, k=1)
            return self.gn(x, sv["ab"], sv["sums"], blk.norm, d_xn, silu=False, resample=RESAMPLE_NONE, add=d_out, add_ld=C)
        dP = P.new((B * heads, T, T), torch.float32, "dP")
        i64 = ctypes.c_int64

        def gemm(A, lda, abs_, ahs, tA, Bm, ldb, bbs, bhs, tB, Cc, ldc, cbs, chs, M, N, K, al=1.0):
            P.call("gemm_batched_simt", A, i64(lda), i64(abs_), i64(ahs), int(tA), Bm, i64(ldb), i64(bbs), i64(bhs), int(tB), Cc,
                   i64(ldc), i64(cbs), i64(chs), M, N, K, B, heads, F32(al), _STREAM)
        # dV = P^T dO
        gemm(probs, T, heads * TT, TT, 1, d_att, C, T * C, ch, 0, d_qkv.at(vo), row, T * row, hs, T, ch, T)
        # dP = dO V^T
        gemm(d_att, C, T * C, ch, 0, qkv.at(vo), row, T * row, hs, 1, dP, T, heads * TT, TT, T, T, ch)
        P.call("softmax_bwd", probs, dP, i64(B * heads * T), T, F32(alpha), _STREAM)   # dS (scale folded in), in place
        # dQ = dS K ; dK = dS^T Q
        gemm(dP, T, heads * TT, TT, 0, qkv.at(ko), row, T * row, hs, 0, d_qkv.at(0), row, T * row, hs, T, ch, T)
        gemm(dP, T, heads * TT, TT, 1, qkv.at(0), row, T * row, hs, 0, d_qkv.at(ko), row, T * row, hs, T, ch, T)
        d_xn = self.conv(sv["xn"], d_qkv, blk.qkv.weight, blk.qkv.bias, B=B, H=H, W=W, Cin=C, Cout=3 * C, k=1)
        return self.gn(x, sv["ab"], sv["sums"], blk.norm, d_xn, silu=False, resample=RESAMPLE_NONE, add=d_out, add_ld=C)

    def head(self, head, sv: dict, d_nchw: Buf) -> Buf:
        P = self.P
        x: Src = sv["x"]
        B, H, W, C = x.B, x.H, x.W, x.C
        conv = head[2]
        Co = conv.weight.shape[0]
        dy = P.new((B, H, W, Co), torch.float32, "d_head")
        P.call("nchw_to_nhwc", d_nchw, dy, B, Co, H * W, _STREAM)
        d_act = self.conv(sv["act"], dy, conv.weight, conv.bias, B=B, H=H, W=W, Cin=C, Cout=Co, k=3)
        return self.gn(x, sv["ab"], sv["sums"], head[0], d_act, silu=True, resample=RESAMPLE_NONE)

    def linear_bank(self, emb_in: Buf, d_bank: Buf, lins: List[nn.Linear], offsets: List[int], total: int, *, B, E,
                    need_dx: bool) -> Optional[Buf]:
        """Backward of  bank = Linear_cat(SiLU(emb_in)) : per-block weight/bias grads, and (optionally) d emb_in."""
        P = self.P
        dw = P.new_grad(E * total)
        self.wgrad_simt(self.fx(emb_in), 0, 1, d_bank, dw, B, 1, 1, E, total, 1, 1, 0)
        db = P.new_grad(total)
        self.colsum(d_bank, B, total, db)
        for lin, off in zip(lins, offsets):
            n = lin.weight.shape[0]
            self.sink.add(lin.weight, dw, E * total, lambda t, off=off, n=n: t.view(E, total)[:, off:off + n].t())
            self.sink.add(lin.bias, db, total, lambda t, off=off, n=n: t[off:off + n])
        if not need_dx:
            return None
        ws = [l.weight for l in lins]
        wt = P.pack(("bank_tco", id(ws[0])), ws, lambda: torch.cat([w.detach() for w in ws], dim=0).float())  # [total][E]
        g = P.new((B, E), torch.float32, "d_silu_emb")
        self.dgrad_simt(d_bank, wt, g, B, 1, 1, E, total, 1, 1, 0)
        dx = P.new((B, E), torch.float32, "d_emb")
        P.call("dsilu_mul", g, self.fx(emb_in), dx, ctypes.c_int64(B * E), _STREAM)
        return dx


# ======================================================================================================================
# ShiftUNet
# ======================================================================================================================

class _Generation:
    """A trainer keeps the saved-for-backward activations in ONE set of plan buffers, so only strictly alternating
    forward / backward is valid.  Each forward stamps a generation; backward refuses to run against buffers that a later
    forward of the same shape has overwritten (two micro-batches before the first backward, retain_graph / double
    backward) instead of returning silently wrong gradients."""
    _gen = 0
    _consumed = -1
    _det_warned = False
    _det_supported = True   # the trainer records deterministic plans under torch.use_deterministic_algorithms

    def _stamp(self) -> int:
        if not self._det_supported and torch.are_deterministic_algorithms_enabled() and not self._det_warned:
            # this trainer keeps its atomic reductions under the switch: say so once, do not raise, so that a training run with
            # the switch on keeps working
            self._det_warned = True
            warnings.warn(f"pdae_b200 {type(self).__name__}: the training forward/backward has no deterministic implementation "
                          "yet; torch.use_deterministic_algorithms covers the pdae_b200 forward-only and sampling paths only",
                          UserWarning, stacklevel=3)
        self._gen += 1
        return self._gen

    def _claim(self, gen: int, what: str) -> None:
        if gen != self._gen:
            raise RuntimeError(f"pdae_b200 {what}: backward for forward call #{gen} but the trainer's activation buffers now "
                               f"hold call #{self._gen} (two forwards of the same shape before the first backward). "
                               "Run forward and backward strictly alternately, or use separate module instances.")
        if self._consumed == gen:
            raise RuntimeError(f"pdae_b200 {what}: backward ran twice for the same forward (retain_graph / double backward "
                               "are not supported by the native backward plans)")
        self._consumed = gen


class ShiftUNetTrainer(_Generation):
    """Forward (fp32, all intermediates kept) + backward plans of a ShiftUNet for one input shape; `amp`: the bf16 plans of
    a forward under autocast (module docstring)."""

    def __init__(self, net, B: int, H: int, W: int, amp: bool = False, det: bool = False):
        from .model.unet import EmbBank, emit_head, emit_stem, emit_time_embed, res_blocks_of
        self.net = net
        self.det = det
        dev = net._device()
        E, base = net.time_embed_dim, net.base_channel
        shift_blocks = res_blocks_of(net.shift_middle_block, net.shift_output_blocks)
        frozen_blocks = res_blocks_of(net.input_blocks, net.middle_block, net.output_blocks)
        # The FROZEN half (input / middle / output blocks, `out` head: 55 % of the forward FLOPs) builds no autograd graph in
        # the reference either (its parameters do not require grad): it runs as a tensor-core plan in the split-operand
        # (fp32-grade) mode -- or, with amp, in the plain "bf16" mode -- with the fused-prologue convs, exactly like sampling;
        # only its skip tensors and bottleneck output are handed to the trainable half.
        self.amp = amp
        Fp = Plan(dev, "bf16" if amp else "bf16x3", deterministic=det)
        self.x_in = Fp.new((B, net.input_channel, H, W), torch.float32, "x_nchw")
        self.t_in = Fp.new((B,), torch.int64, "t")
        self.x_in.keep = self.t_in.keep = True
        emb_f = emit_time_embed(Fp, net.time_embed, self.t_in, B, base, E, dev)
        bank_f = EmbBank(Fp, frozen_blocks, "t", emb_f, B, E, "train_t_frozen")
        hf = emit_stem(Fp, net.input_blocks[0][0], self.x_in, B, H, W, net.input_channel)
        hs_f = [hf]
        for stage in list(net.input_blocks)[1:]:
            hf = stage.emit(Fp, hf, bank_f)
            hs_f.append(hf)
        skips = []                             # consumed by the trainable half's plan: private storage
        for sfrc in hs_f:
            b = sfrc.b1
            if b.dtype != torch.float32:       # bf16 residual stream (amp): widened to fp32 once per step
                b, _ = Fp.gn_apply(b, sfrc.C, None, 0, None, silu=False, resample=RESAMPLE_NONE, B=B, H=sfrc.H, W=sfrc.W,
                                   act_dtype=torch.float32)
            b.keep = True
            skips.append((b, sfrc))
        eps_h = net.middle_block.emit(Fp, hf, bank_f)
        for stage, skip in zip(net.output_blocks, reversed(hs_f)):
            eps_h = stage.emit(Fp, eps_h.cat(skip), bank_f)
        self.eps = Fp.new((B, net.output_channel, H, W), torch.float32, "eps_nchw")
        self.eps.keep = True
        emit_head(Fp, net.out, eps_h, self.eps)
        Fp.finalize()
        self.frozen = Fp
        P = Plan(dev, "fp32", deterministic=det)
        P.keep_all = True
        P.train_tc = "bf16" if amp else "bf16x3"   # trainable half: fp32 activations kept, convs on the tensor cores
        self.z_in = P.new((B, net.latent_dim), torch.float32, "z")
        emb = emit_time_embed(P, net.time_embed, P.fixed(self.t_in.tensor), B, base, E, dev)
        shift_emb = P.new((B, E), torch.float32, "shift_emb")
        P.linear(self.z_in, net.label_emb.weight, net.label_emb.bias, shift_emb, B=B, Cin=net.latent_dim, Cout=E)
        bank_t = EmbBank(P, shift_blocks, "t", emb, B, E, "train_t_shift")
        bank_z = EmbBank(P, shift_blocks, "z", shift_emb, B, E, "train_z_shift")
        tape: list = []
        hs = [Src(P.fixed(b.tensor), sfrc.C, B, sfrc.H, sfrc.W) for b, sfrc in skips]
        shift_h = net.shift_middle_block.emit(P, hs[-1], bank_t, bank_z, tape=tape)
        for shift_stage in net.shift_output_blocks:
            shift_h = shift_stage.emit(P, shift_h.cat(hs.pop()), bank_t, bank_z, tape=tape)
        self.grad = P.new((B, net.input_channel, H, W), torch.float32, "shift_nchw")
        emit_head(P, net.shift_out, shift_h, self.grad, tape=tape)
        P.finalize()
        self.fwd = P

        # ---------------- backward plan ----------------
        BP = bwd_plan(dev, amp, det)
        self.sink = GradSink()
        bw = Backward(BP, self.sink)
        self.d_grad = BP.new((B, net.input_channel, H, W), torch.float32, "d_shift_nchw")
        self.d_grad.keep = True
        d_bank_t = BP.new((B, bank_t.total), torch.float32, "d_bank_t")
        d_bank_z = BP.new((B, bank_z.total), torch.float32, "d_bank_z")
        d = None
        for kind, mod, sv in reversed(tape):
            if kind == "head":
                d = bw.head(mod, sv, self.d_grad)
            elif kind == "res":
                d = bw.resblock(mod, sv, d, (d_bank_t, bank_t.offsets[id(mod)], bank_t.total),
                                (d_bank_z, bank_z.offsets[id(mod)], bank_z.total))
            else:
                d = bw.attention(mod, sv, d)
        # d now = grad wrt the (frozen) middle input: not needed.  Embedding paths:
        lt = [b.emb_layers[1] for b in shift_blocks]
        lz = [b.emb_z_layers[1] for b in shift_blocks]
        bw.linear_bank(emb, d_bank_t, lt, [bank_t.offsets[id(b)] for b in shift_blocks], bank_t.total, B=B, E=E, need_dx=False)
        d_shift_emb = bw.linear_bank(shift_emb, d_bank_z, lz, [bank_z.offsets[id(b)] for b in shift_blocks], bank_z.total, B=B,
                                     E=E, need_dx=True)
        self.dz = bw.conv(self.z_in, d_shift_emb, net.label_emb.weight, net.label_emb.bias, B=B, H=1, W=1, Cin=net.latent_dim,
                          Cout=E, k=1, w_unpack=lambda t, L=net.latent_dim: t.view(L, E).t())
        self.dz.keep = True
        BP.finalize()
        self.bwd = BP
        self.params = [p for m in net._shift_parts() for p in m.parameters()]

    def stale(self) -> bool:
        return self.fwd.stale() or self.bwd.stale() or self.frozen.stale()

    def forward(self, x, t, z):
        draw_dropout_masks(self.fwd)
        self.x_in.tensor.copy_(x)
        self.t_in.tensor.copy_(t)
        self.z_in.tensor.copy_(z)
        self.frozen.run()
        self.fwd.run()
        return self.eps.tensor.clone(), self.grad.tensor.clone()

    def backward(self, d_grad):
        self.d_grad.tensor.copy_(d_grad)
        self.bwd.run()
        grads = self.sink.collect()
        return self.dz.tensor.reshape(self.z_in.shape).clone(), [grads.get(id(p)) for p in self.params]


class _ShiftUNetFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, trainer: ShiftUNetTrainer, x, t, z, *params):
        ctx.trainer = trainer
        ctx.gen = trainer._stamp()
        ctx.z_needs = z.requires_grad
        with torch.no_grad():
            eps, grad = trainer.forward(x, t, z)
        ctx.mark_non_differentiable(eps)
        return eps, grad

    @staticmethod
    def backward(ctx, d_eps, d_grad):
        tr = ctx.trainer
        tr._claim(ctx.gen, "ShiftUNet")
        with torch.no_grad():
            dz, pgrads = tr.backward(d_grad.contiguous())
        return (None, None, None, dz if ctx.z_needs else None, *pgrads)


def shiftunet_train_forward(net, x, t, z):
    B, C, H, W = x.shape
    amp = autocast_active()
    det = torch.are_deterministic_algorithms_enabled()
    key = ("train", B, H, W, tuple(m.training for m in net._shift_parts()), amp, det)
    cache = net.__dict__.setdefault("_train_cache", {})
    tr = cache.get(key)
    if tr is None or tr.stale():
        tr = ShiftUNetTrainer(net, B, H, W, amp, det)
        cache[key] = tr
    return _ShiftUNetFn.apply(tr, x, t, z, *tr.params)


# ======================================================================================================================
# Plain UNet (regular DPM training, gaussian_diffusion.py:199-211) -- every parameter trainable, skip gradients routed
# ======================================================================================================================
class UNetTrainer(_Generation):
    def __init__(self, net, B: int, H: int, W: int, amp: bool = False, det: bool = False):
        from .model.unet import EmbBank, emit_head, res_blocks_of
        from .model.module import timestep_freqs
        self.net = net
        self.amp = amp
        self.det = det
        dev = net._device()
        P = Plan(dev, "fp32", deterministic=det)
        P.keep_all = True
        P.train_tc = "bf16" if amp else "bf16x3"   # convs on the tensor cores, fp32 activations kept
        E, base, Cimg = net.time_embed_dim, net.base_channel, net.input_channel
        self.x_in = P.new((B, Cimg, H, W), torch.float32, "x_nchw")
        self.t_in = P.new((B,), torch.int64, "t")
        self.c_in = P.new((B,), torch.int64, "cond") if net.num_class is not None else None
        te = net.time_embed
        temb = P.new((B, base), torch.float32, "temb")
        P.call("timestep_embedding", self.t_in, B, base, P.fixed(timestep_freqs(base, dev)), temb, _STREAM)
        th = P.new((B, E), torch.float32, "temb_h")
        P.linear(temb, te[0].weight, te[0].bias, th, B=B, Cin=base, Cout=E)
        emb = P.new((B, E), torch.float32, "emb")
        P.linear(th, te[2].weight, te[2].bias, emb, B=B, Cin=E, Cout=E, a_silu=True)
        if self.c_in is not None:
            P.call("embedding_add", emb, P.param(net.label_emb.weight), self.c_in, B, E, _STREAM)
        blocks = res_blocks_of(net.input_blocks, net.middle_block, net.output_blocks)
        bank = EmbBank(P, blocks, "t", emb, B, E, "train_unet_t")
        stem = net.input_blocks[0][0]
        c0 = stem.weight.shape[0]
        h0 = P.new((B, H, W, c0), torch.float32, "stem")
        P.conv(self.x_in, stem.weight, stem.bias, h0, B=B, H=H, W=W, Cin=Cimg, Cout=c0, k=3, in_nchw=True)
        h = Src(h0, c0, B, H, W)
        hs = [h]
        enc_tapes = []
        for stage in list(net.input_blocks)[1:]:
            tp: list = []
            h = stage.emit(P, h, bank, tape=tp)
            enc_tapes.append(tp)
            hs.append(h)
        mid_tape: list = []
        h = net.middle_block.emit(P, h, bank, tape=mid_tape)
        dec_tapes = []
        n_skip = len(hs)
        for stage in net.output_blocks:
            tp = []
            h = stage.emit(P, h.cat(hs.pop()), bank, tape=tp)
            dec_tapes.append(tp)
        self.out = P.new((B, net.output_channel, H, W), torch.float32, "eps_nchw")
        head_tape: list = []
        emit_head(P, net.out, h, self.out, tape=head_tape)
        P.finalize()
        self.fwd = P

        BP = bwd_plan(dev, amp, det)
        self.sink = GradSink()
        bw = Backward(BP, self.sink)
        self.d_out = BP.new((B, net.output_channel, H, W), torch.float32, "d_eps_nchw")
        self.d_out.keep = True
        d_bank = BP.new((B, bank.total), torch.float32, "d_bank_t")
        slot = lambda mod: (d_bank, bank.offsets[id(mod)], bank.total)

        def run_tape(tp, d, first_has_skip):
            dskip = None
            for li, (kind, mod, sv) in reversed(list(enumerate(tp))):
                if kind == "res":
                    if li == 0 and first_has_skip:
                        d, dskip = bw.resblock(mod, sv, d, slot(mod), None, want_dx2=True)
                    else:
                        d = bw.resblock(mod, sv, d, slot(mod), None)
                else:
                    d = bw.attention(mod, sv, d)
            return d, dskip

        d = bw.head(net.out, head_tape[0][2], self.d_out)
        dskips = [None] * n_skip
        for j in reversed(range(len(dec_tapes))):
            d, dsk = run_tape(dec_tapes[j], d, True)
            dskips[n_skip - 1 - j] = dsk       # decoder stage j consumed hs[n_skip-1-j]
        d, _ = run_tape(mid_tape, d, False)
        for i in reversed(range(len(enc_tapes))):          # encoder stage i produced hs[i+1]
            sk = dskips[i + 1]
            BP.call("add_inplace", d, sk, ctypes.c_int64(sk.nbytes // 4), _STREAM)
            d, _ = run_tape(enc_tapes[i], d, False)
        BP.call("add_inplace", d, dskips[0], ctypes.c_int64(dskips[0].nbytes // 4), _STREAM)
        bw.conv(self.x_in, d, stem.weight, stem.bias, B=B, H=H, W=W, Cin=Cimg, Cout=c0, k=3, need_dx=False, in_nchw=True)
        # embedding path: d emb -> (label_emb) -> time_embed MLP
        lins = [b.emb_layers[1] for b in blocks]
        d_emb = bw.linear_bank(emb, d_bank, lins, [bank.offsets[id(b)] for b in blocks], bank.total, B=B, E=E, need_dx=True)
        if self.c_in is not None:
            dwl = BP.new_grad(net.label_emb.weight.numel())
            if det:
                BP.call("embedding_bwd_det", d_emb, bw.fx(self.c_in), dwl, B, E, net.label_emb.weight.shape[0], _STREAM)
            else:
                BP.call("embedding_bwd", d_emb, bw.fx(self.c_in), dwl, B, E, _STREAM)
            self.sink.add(net.label_emb.weight, dwl, net.label_emb.weight.numel(), lambda t: t)
        # emb = Linear2(SiLU(th)) ; th = Linear0(temb)
        d_sth = bw.conv(th, d_emb, te[2].weight, te[2].bias, B=B, H=1, W=1, Cin=E, Cout=E, k=1, a_silu=True,
                        w_unpack=lambda t: t.view(E, E).t())
        d_th = BP.new((B, E), torch.float32, "d_th")
        BP.call("dsilu_mul", d_sth, bw.fx(th), d_th, ctypes.c_int64(B * E), _STREAM)
        bw.conv(temb, d_th, te[0].weight, te[0].bias, B=B, H=1, W=1, Cin=base, Cout=E, k=1, need_dx=False,
                w_unpack=lambda t: t.view(base, E).t())
        BP.finalize()
        self.bwd = BP
        self.params = [p for p in net.parameters()]

    def forward(self, x, t, cond):
        draw_dropout_masks(self.fwd)
        self.x_in.tensor.copy_(x)
        self.t_in.tensor.copy_(t)
        if self.c_in is not None:
            self.c_in.tensor.copy_(cond)
        self.fwd.run()
        return self.out.tensor.clone()

    def backward(self, d_out):
        self.d_out.tensor.copy_(d_out)
        self.bwd.run()
        grads = self.sink.collect()
        return [grads.get(id(p)) for p in self.params]


class _UNetFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, trainer: UNetTrainer, x, t, cond, *params):
        ctx.trainer = trainer
        ctx.gen = trainer._stamp()
        with torch.no_grad():
            return trainer.forward(x, t, cond)

    @staticmethod
    def backward(ctx, d_out):
        ctx.trainer._claim(ctx.gen, "UNet")
        with torch.no_grad():
            pg = ctx.trainer.backward(d_out.contiguous())
        return (None, None, None, None, *pg)


def unet_train_forward(net, x, t, cond):
    B, C, H, W = x.shape
    cache = net.__dict__.setdefault("_train_cache", {})
    amp = autocast_active()
    det = torch.are_deterministic_algorithms_enabled()
    key = (B, H, W, net.training, amp, det)
    tr = cache.get(key)
    if tr is None or tr.fwd.stale() or tr.bwd.stale():
        tr = UNetTrainer(net, B, H, W, amp, det)
        cache[key] = tr
    return _UNetFn.apply(tr, x, t, cond, *tr.params)


# ======================================================================================================================
# Semantic encoder
# ======================================================================================================================
class EncoderTrainer(_Generation):
    """Forward (fp32, all intermediates kept) + backward plans of a semantic encoder for one input shape; `amp`: the bf16
    plans of a forward under autocast -- its stride-2 and attention convs, their data and weight gradients run as single-pass
    bf16 MMAs (the 3-channel stem and the final Linear stay on CUDA cores)."""

    def __init__(self, enc, B: int, H: int, W: int, amp: bool = False, det: bool = False):
        self.enc = enc
        self.amp = amp
        self.det = det
        dev = enc._device()
        P = Plan(dev, "fp32", deterministic=det)
        P.keep_all = True
        if amp:
            P.train_tc = "bf16"
        self.x_in = P.new((B, 3, H, W), torch.float32, "x_nchw")
        tape = []          # ("conv", mod, dict) / ("attn", ...) / ("fc", ...)
        h: Optional[Src] = None
        C = 3
        pend = None        # (ab, sums, gn module) of the GN whose SiLU output feeds the next conv / fc
        self.z = None
        for kind, idx in enc._order:
            m = enc.encoder[idx]
            if kind == "conv":
                Co = m.weight.shape[0]
                Ho, Wo = H // 2, W // 2
                out = P.new((B, Ho, Wo, Co), torch.float32, "enc_h")
                if h is None:
                    P.conv(self.x_in, m.weight, m.bias, out, B=B, H=H, W=W, Cin=3, Cout=Co, k=3, stride=2, pad=1, in_nchw=True)
                    tape.append(("conv", m, dict(x=None, act=self.x_in, nchw=True, B=B, H=H, W=W, Cin=3, Cout=Co, gn=None)))
                else:
                    act, _ = P.gn_apply(h.b1, C, None, 0, pend[0], silu=True, resample=RESAMPLE_NONE, B=B, H=H, W=W,
                                        act_dtype=torch.float32)
                    P.conv(act, m.weight, m.bias, out, B=B, H=H, W=W, Cin=C, Cout=Co, k=3, stride=2, pad=1)
                    tape.append(("conv", m, dict(x=h, act=act, nchw=False, B=B, H=H, W=W, Cin=C, Cout=Co, gn=pend)))
                h, C, H, W = Src(out, Co, B, Ho, Wo), Co, Ho, Wo
            elif kind == "gn":
                ab = P.gn_coef(h.b1, C, None, 0, m.weight, m.bias, B=B, HW=H * W)
                pend = (ab, P.last_sums, m)
            elif kind == "attn":
                h = m.emit(P, h, tape=tape)
            else:
                act, _ = P.gn_apply(h.b1, C, None, 0, pend[0], silu=True, resample=RESAMPLE_NONE, B=B, H=H, W=W,
                                    act_dtype=torch.float32)
                wt, HW = m.weight, H * W
                wp = P.pack((id(wt), "enc_fc"), [wt],
                            lambda: wt.detach().reshape(-1, C, HW).permute(2, 1, 0).reshape(HW * C, -1).float())
                self.z = P.new((B, enc.latent_dim), torch.float32, "z")
                P.linear_packed(act, wp, P.param(m.bias), self.z, B=B, Cin=HW * C, Cout=enc.latent_dim)
                tape.append(("fc", m, dict(x=h, act=act, gn=pend, B=B, H=H, W=W, C=C)))
        P.finalize()
        self.fwd = P

        BP = bwd_plan(dev, amp, det)
        self.sink = GradSink()
        bw = Backward(BP, self.sink)
        L = enc.latent_dim
        self.dz = BP.new((B, L), torch.float32, "dz")
        self.dz.keep = True
        d = self.dz
        for kind, m, sv in reversed(tape):
            if kind == "fc":
                Bc, Hh, Ww, Cc = sv["B"], sv["H"], sv["W"], sv["C"]
                HW = Hh * Ww
                K = HW * Cc
                dw = BP.new_grad(K * L)
                bw.wgrad_simt(bw.fx(sv["act"]), 0, 0, d, dw, Bc, 1, 1, K, L, 1, 1, 0)
                # packed [HW*C][L] (NHWC flatten) -> reference layout [L][C*HW] (NCHW flatten)
                self.sink.add(m.weight, dw, K * L, lambda t, HW=HW, Cc=Cc: t.view(HW, Cc, L).permute(2, 1, 0))
                db = BP.new_grad(L)
                bw.colsum(d, Bc, L, db)
                self.sink.add(m.bias, db, L, lambda t: t)
                wt = m.weight
                wtco = BP.pack((id(wt), "enc_fc_tco"), [wt],
                               lambda: wt.detach().reshape(L, Cc, HW).permute(0, 2, 1).reshape(L, HW * Cc).float())
                d_act = BP.new((Bc, Hh, Ww, Cc), torch.float32, "d_fc_in")
                bw.dgrad_simt(d, wtco, d_act, Bc, 1, 1, K, L, 1, 1, 0)
                ab, sums, gnm = sv["gn"]
                d = bw.gn(sv["x"], ab, sums, gnm, d_act, silu=True, resample=RESAMPLE_NONE)
            elif kind == "attn":
                d = bw.attention(m, sv, d)
            else:
                first = sv["x"] is None
                d_act = bw.conv(sv["act"], d, m.weight, m.bias, B=sv["B"], H=sv["H"], W=sv["W"], Cin=sv["Cin"], Cout=sv["Cout"],
                                k=3, stride=2, pad=1, need_dx=not first, in_nchw=sv["nchw"])
                if not first:
                    ab, sums, gnm = sv["gn"]
                    d = bw.gn(sv["x"], ab, sums, gnm, d_act, silu=True, resample=RESAMPLE_NONE)
        BP.finalize()
        self.bwd = BP
        self.params = list(enc.parameters())

    def forward(self, x):
        self.x_in.tensor.copy_(x)
        self.fwd.run()
        return self.z.tensor.clone()

    def backward(self, dz):
        self.dz.tensor.copy_(dz)
        self.bwd.run()
        grads = self.sink.collect()
        return [grads.get(id(p)) for p in self.params]


class _EncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, trainer: EncoderTrainer, x, *params):
        ctx.trainer = trainer
        ctx.gen = trainer._stamp()
        with torch.no_grad():
            return trainer.forward(x)

    @staticmethod
    def backward(ctx, dz):
        ctx.trainer._claim(ctx.gen, "encoder")
        with torch.no_grad():
            pg = ctx.trainer.backward(dz.contiguous())
        return (None, None, *pg)


def encoder_train_forward(enc, x):
    B, C, H, W = x.shape
    cache = enc.__dict__.setdefault("_train_cache", {})
    amp = autocast_active()
    det = torch.are_deterministic_algorithms_enabled()
    key = (B, H, W, amp, det)
    tr = cache.get(key)
    if tr is None or tr.fwd.stale() or tr.bwd.stale():
        tr = EncoderTrainer(enc, B, H, W, amp, det)
        cache[key] = tr
    return _EncoderFn.apply(tr, x, *tr.params)


# ======================================================================================================================
# MLPSkipNet (latent DPM training, diffusion/gaussian_diffusion.py:373-398)
# ======================================================================================================================
def mlp_amp_supported(net) -> bool:
    """Every Linear of the MLPSkipNet except time_embed has Cin and Cout in {D, Wd, Wd + D}: multiples of 64 put them all on
    the tensor cores, which the bf16 trainer needs."""
    return net.input_channel % 64 == 0 and net.model_channel % 64 == 0 and len(net.layers) >= 2


def _tensor_of(b, shape) -> torch.Tensor:
    """The tensor behind a plan buffer or a view of one (a split-K output lives in the plan's zeroed arena)."""
    if isinstance(b, BufView):
        return b.buf.tensor[b.off: b.off + int(np.prod(shape))].view(shape)
    return b.tensor


class MLPTrainer(_Generation):
    """Forward plan keeping every layer's (input, pre-activation, modulation) + backward plan for all parameters of the
    MLPSkipNet; no gradient w.r.t. z_t (the reference's z_t is built from detached latents).  `amp`: the bf16 plans of a
    forward under autocast (_init_amp).  Its LayerNorm / split-K reductions have no deterministic form yet."""
    _det_supported = False

    def __init__(self, net, B: int, amp: bool = False):
        self.net = net
        self.amp = amp
        self.B = B
        if amp:
            self._init_amp(net, B)
            return
        dev = net._device()
        D, Wd, Te = net.input_channel, net.model_channel, net.time_emb_channel
        from .model.module import timestep_freqs
        P = Plan(dev, "fp32")
        P.keep_all = True
        self.x_in = P.new((B, D), torch.float32, "z_t")
        self.t_in = P.new((B,), torch.int64, "t")
        temb = P.new((B, Te), torch.float32, "temb")
        P.call("timestep_embedding", self.t_in, B, Te, P.fixed(timestep_freqs(Te, dev)), temb, _STREAM)
        c0 = P.new((B, D), torch.float32, "cond_h")
        P.linear(temb, net.time_embed[0].weight, net.time_embed[0].bias, c0, B=B, Cin=Te, Cout=D)
        cond = P.new((B, D), torch.float32, "cond")
        P.linear(c0, net.time_embed[2].weight, net.time_embed[2].bias, cond, B=B, Cin=D, Cout=D, a_silu=True)
        scond = P.new((B, D), torch.float32, "silu_cond")    # SiLU(cond): the input of every linear_emb
        P.call("mlp_mod_ln_act", cond, None, None, None, F32(1e-5), 1, scond, D, B, D, _STREAM)
        cur, cin = self.x_in, D
        n = len(net.layers)
        tape = []
        for i, layer in enumerate(net.layers):
            last = i == n - 1
            co = layer.linear.weight.shape[0]
            h = P.new((B, co), torch.float32, "mlp_h")
            P.linear(cur, layer.linear.weight, layer.linear.bias, h, B=B, Cin=cin, Cout=co)
            if last:
                self.out = h
                tape.append(dict(layer=layer, x=cur, cin=cin, co=co, last=True))
                break
            cnd = P.new((B, co), torch.float32, "mlp_cond")
            P.linear(scond, layer.linear_emb.weight, layer.linear_emb.bias, cnd, B=B, Cin=D, Cout=co)
            dst = P.new((B, Wd + D), torch.float32, f"cat{i}")   # one concat buffer per layer: the backward reads them all
            P.call("copy_cols", self.x_in, dst, Wd + D, Wd, B, D, _STREAM)
            ln = layer.norm if isinstance(layer.norm, nn.LayerNorm) else None
            P.call("mlp_mod_ln_act", h, cnd, P.param(ln.weight) if ln else None, P.param(ln.bias) if ln else None,
                   F32(ln.eps if ln else 1e-5), 1, dst, Wd + D, B, co, _STREAM)
            mask = None
            pdrop = float(layer.dropout.p) if isinstance(layer.dropout, nn.Dropout) else 0.0
            if net.training and pdrop > 0:
                mask = P.new((B, co), torch.float32, "drop_mask")
                P.dropout_masks.append((layer, mask, pdrop))
                P.call("mul_mask_cols", dst, Wd + D, mask, F32(1.0 / (1.0 - pdrop)), B, co, _STREAM)
            tape.append(dict(layer=layer, x=cur, cin=cin, co=co, last=False, h=h, cnd=cnd, ln=ln, mask=mask, pdrop=pdrop))
            cur, cin = dst, Wd + D
        P.finalize()
        self.fwd = P

        BP = bwd_plan(dev)
        self.sink = GradSink()
        bw = Backward(BP, self.sink)
        self.d_out = BP.new((B, D), torch.float32, "d_eps")
        self.d_out.keep = True
        d_scond = BP.new_zeroed(B * D)          # sum over layers of d SiLU(cond)
        dy, dy_ld = self.d_out, D
        for sv in reversed(tape):
            layer, co, cin = sv["layer"], sv["co"], sv["cin"]
            if sv["last"]:
                dh = dy
            else:
                if sv["mask"] is not None:
                    BP.call("mul_mask_cols", dy, dy_ld, bw.fx(sv["mask"]), F32(1.0 / (1.0 - sv["pdrop"])), B, co, _STREAM)
                ln = sv["ln"]
                dlw = dlb = None
                if ln is not None:
                    dlw, dlb = BP.new_zeroed(co), BP.new_zeroed(co)
                    self.sink.add(ln.weight, dlw, co, lambda t: t)
                    self.sink.add(ln.bias, dlb, co, lambda t: t)
                dh = BP.new((B, co), torch.float32, "d_mlp_h")
                dcnd = BP.new((B, co), torch.float32, "d_mlp_cond")
                BP.call("mlp_mod_ln_act_bwd", bw.fx(sv["h"]), bw.fx(sv["cnd"]), BP.param(ln.weight) if ln else None,
                        BP.param(ln.bias) if ln else None, F32(ln.eps if ln else 1e-5), 1, dy, dy_ld, dh, dcnd, dlw, dlb, B, co,
                        _STREAM)
                g = bw.conv(scond, dcnd, layer.linear_emb.weight, layer.linear_emb.bias, B=B, H=1, W=1, Cin=D, Cout=co, k=1)
                BP.call("add_inplace", d_scond, g, ctypes.c_int64(B * D), _STREAM)
            first = sv["x"] is self.x_in
            dx = bw.conv(sv["x"], dh, layer.linear.weight, layer.linear.bias, B=B, H=1, W=1, Cin=cin, Cout=co, k=1,
                         need_dx=not first)
            if not first:
                dy, dy_ld = dx, cin                       # left Wd columns = grad of the previous layer's activation
        d_cond = BP.new((B, D), torch.float32, "d_cond")
        BP.call("dsilu_mul", d_scond, bw.fx(cond), d_cond, ctypes.c_int64(B * D), _STREAM)
        g = bw.conv(c0, d_cond, net.time_embed[2].weight, net.time_embed[2].bias, B=B, H=1, W=1, Cin=D, Cout=D, k=1, a_silu=True)
        d_c0 = BP.new((B, D), torch.float32, "d_c0")
        BP.call("dsilu_mul", g, bw.fx(c0), d_c0, ctypes.c_int64(B * D), _STREAM)
        bw.conv(temb, d_c0, net.time_embed[0].weight, net.time_embed[0].bias, B=B, H=1, W=1, Cin=Te, Cout=D, k=1, need_dx=False)
        BP.finalize()
        self.bwd = BP
        self.params = [p for p in net.parameters() if p.requires_grad]

    def _init_amp(self, net, B: int) -> None:
        """bf16 plans (the reference's enable_amp): every Linear except time_embed is one bf16 MMA per product with fp32
        accumulation and fp32 output, split-K where its output tiles alone would leave SMs idle (Plan.linear_tc).  The
        layers' linear_emb, which all read SiLU(cond), are one bank GEMM over their concatenated weights, forward and
        backward.  Modulate, LayerNorm, SiLU and dropout write the next Linear's bf16 operand straight into a bf16 concat
        buffer (pdae_mlp_mod_ln_act_bf16), which the weight gradient reads again; h and the bank output stay fp32 for the
        backward, which writes fp32 and bf16 gradients in one pass (pdae_mlp_mod_ln_act_bwd_bf16).  time_embed (64 -> 512,
        SiLU, 512 -> 512) stays fp32 on CUDA cores in the forward."""
        dev = net._device()
        D, Wd, Te = net.input_channel, net.model_channel, net.time_emb_channel
        from .model.module import timestep_freqs
        bf16 = torch.bfloat16
        P = Plan(dev, "fp32")
        P.keep_all = True
        self.x_in = P.new((B, D), torch.float32, "z_t")
        self.t_in = P.new((B,), torch.int64, "t")
        temb = P.new((B, Te), torch.float32, "temb")
        P.call("timestep_embedding", self.t_in, B, Te, P.fixed(timestep_freqs(Te, dev)), temb, _STREAM)
        c0 = P.new((B, D), torch.float32, "cond_h")
        P.linear(temb, net.time_embed[0].weight, net.time_embed[0].bias, c0, B=B, Cin=Te, Cout=D)
        cond = P.new((B, D), torch.float32, "cond")
        P.linear(c0, net.time_embed[2].weight, net.time_embed[2].bias, cond, B=B, Cin=D, Cout=D, a_silu=True)
        scond = P.new((B, D), bf16, "silu_cond_bf16")     # SiLU(cond): the operand of the bank GEMM
        P.call("mlp_mod_ln_act_bf16", cond, None, 0, None, None, F32(1e-5), 1, None, F32(1.0), scond, D, B, D, _STREAM)
        # the bank: linear_emb of every conditioned layer, [total][D] weights / [total] bias, layer i at column offsets[i]
        emb_layers = [layer for layer in net.layers if layer.use_cond]
        ws, bs = [l.linear_emb.weight for l in emb_layers], [l.linear_emb.bias for l in emb_layers]
        offsets = np.cumsum([0] + [w.shape[0] for w in ws]).tolist()
        total = offsets[-1]
        for p in ws + bs:
            P.params.append((p, p.data_ptr()))
        wbank = P.pack(("mlp_bank", id(ws[0])), ws, lambda: torch.cat([w.detach() for w in ws], 0).to(bf16))
        bbank = P.pack(("mlp_bank_bias", id(bs[0])), bs, lambda: torch.cat([b.detach() for b in bs]).float())
        bank = P.linear_tc(scond, wbank, bbank, B=B, Cin=D, Cout=total, name="mlp_bank")
        x_bf = P.new((B, D), bf16, "z_t_bf16")
        P.call("copy_cols_bf16", self.x_in, x_bf, D, 0, B, D, _STREAM)
        cur, cin = x_bf, D
        n = len(net.layers)
        tape = []
        for i, layer in enumerate(net.layers):
            co = layer.linear.weight.shape[0]
            w = layer.linear.weight
            wp = P.pack((id(w), "tc"), [w], lambda w=w: w.detach().to(bf16))
            h = P.linear_tc(cur, wp, P.param(layer.linear.bias), B=B, Cin=cin, Cout=co, name="mlp_h")
            if i == n - 1:
                self.out = h
                tape.append(dict(layer=layer, x=cur, cin=cin, co=co, last=True))
                break
            off = offsets[emb_layers.index(layer)]
            dst = P.new((B, Wd + D), bf16, f"cat{i}")    # one bf16 concat buffer per layer: the weight gradients read them all
            P.call("copy_cols_bf16", self.x_in, dst, Wd + D, Wd, B, D, _STREAM)
            ln = layer.norm if isinstance(layer.norm, nn.LayerNorm) else None
            mask = None
            pdrop = float(layer.dropout.p) if isinstance(layer.dropout, nn.Dropout) else 0.0
            if net.training and pdrop > 0:
                mask = P.new((B, co), torch.float32, "drop_mask")
                P.dropout_masks.append((layer, mask, pdrop))
            P.call("mlp_mod_ln_act_bf16", h, bank.at(off), total, P.param(ln.weight) if ln else None,
                   P.param(ln.bias) if ln else None, F32(ln.eps if ln else 1e-5), 1, mask,
                   F32(1.0 / (1.0 - pdrop) if mask is not None else 1.0), dst, Wd + D, B, co, _STREAM)
            tape.append(dict(layer=layer, x=cur, cin=cin, co=co, last=False, h=h, off=off, ln=ln, mask=mask, pdrop=pdrop))
            cur, cin = dst, Wd + D
        P.finalize()
        self.fwd = P

        BP = bwd_plan(dev, amp=True)
        self.sink = GradSink()
        bw = Backward(BP, self.sink)
        self.d_out = BP.new((B, D), torch.float32, "d_eps")
        self.d_out.keep = True
        d_bank = BP.new((B, total), torch.float32, "d_bank")        # every column block written by its layer's kernel
        d_bank_bf = BP.new((B, total), bf16, "d_bank_bf16")
        dy, dy_ld = self.d_out, D
        for sv in reversed(tape):
            layer, co, cin = sv["layer"], sv["co"], sv["cin"]
            w = layer.linear.weight
            if sv["last"]:
                dh = dy
                dh_bf = BP.new((B, co), bf16, "d_mlp_h_bf16")
                BP.call("copy_cols_bf16", dy, dh_bf, co, 0, B, co, _STREAM)
            else:
                ln = sv["ln"]
                dlw = dlb = None
                if ln is not None:
                    dlw, dlb = BP.new_zeroed(co), BP.new_zeroed(co)
                    self.sink.add(ln.weight, dlw, co, lambda t: t)
                    self.sink.add(ln.bias, dlb, co, lambda t: t)
                dh = BP.new((B, co), torch.float32, "d_mlp_h")
                dh_bf = BP.new((B, co), bf16, "d_mlp_h_bf16")
                mask = sv["mask"]
                BP.call("mlp_mod_ln_act_bwd_bf16", bw.fx(sv["h"]), bw.fx(bank).at(sv["off"]), total,
                        BP.param(ln.weight) if ln else None, BP.param(ln.bias) if ln else None, F32(ln.eps if ln else 1e-5), 1,
                        dy, dy_ld, bw.fx(mask), F32(1.0 / (1.0 - sv["pdrop"]) if mask is not None else 1.0), dh, dh_bf,
                        d_bank.at(sv["off"]), d_bank_bf.at(sv["off"]), dlw, dlb, B, co, _STREAM)
            dw = BP.new_zeroed(cin * co)
            BP.call("wgrad_tc_bf16", bw.fx(sv["x"]), dh_bf, dw, B, 1, 1, cin, co, 1, flops=2.0 * B * cin * co)
            self.sink.add(w, dw, cin * co, lambda t, cin=cin, co=co: t.view(cin, co).t())
            db = BP.new_zeroed(co)
            BP.call("colsum", dh, ctypes.c_int64(B), co, db, _STREAM)
            self.sink.add(layer.linear.bias, db, co, lambda t: t)
            if sv["x"] is not x_bf:                       # (no gradient w.r.t. z_t)
                wt = BP.pack((id(w), "tc_t"), [w], lambda w=w: w.detach().t().contiguous().to(bf16))     # [cin][co]
                dy, dy_ld = BP.linear_tc(dh_bf, wt, None, B=B, Cin=co, Cout=cin, name="d_mlp_x"), cin
        # the bank: one weight gradient, one bias column sum, one data gradient for all conditioned layers
        dwb = BP.new_zeroed(D * total)
        BP.call("wgrad_tc_bf16", bw.fx(scond), d_bank_bf, dwb, B, 1, 1, D, total, 1, flops=2.0 * B * D * total)
        dbb = BP.new_zeroed(total)
        BP.call("colsum", d_bank, ctypes.c_int64(B), total, dbb, _STREAM)
        for layer, off in zip(emb_layers, offsets):
            co = layer.linear_emb.weight.shape[0]
            self.sink.add(layer.linear_emb.weight, dwb, D * total, lambda t, off=off, co=co: t.view(D, total)[:, off:off + co].t())
            self.sink.add(layer.linear_emb.bias, dbb, total, lambda t, off=off, co=co: t[off:off + co])
        wbt = BP.pack(("mlp_bank_t", id(ws[0])), ws, lambda: torch.cat([w.detach() for w in ws], 0).t().contiguous().to(bf16))
        d_scond = BP.linear_tc(d_bank_bf, wbt, None, B=B, Cin=total, Cout=D, name="d_silu_cond")
        d_cond = BP.new((B, D), torch.float32, "d_cond")
        BP.call("dsilu_mul", d_scond, bw.fx(cond), d_cond, ctypes.c_int64(B * D), _STREAM)
        g = bw.conv(c0, d_cond, net.time_embed[2].weight, net.time_embed[2].bias, B=B, H=1, W=1, Cin=D, Cout=D, k=1, a_silu=True)
        d_c0 = BP.new((B, D), torch.float32, "d_c0")
        BP.call("dsilu_mul", g, bw.fx(c0), d_c0, ctypes.c_int64(B * D), _STREAM)
        bw.conv(temb, d_c0, net.time_embed[0].weight, net.time_embed[0].bias, B=B, H=1, W=1, Cin=Te, Cout=D, k=1, need_dx=False)
        BP.finalize()
        self.bwd = BP
        self.params = [p for p in net.parameters() if p.requires_grad]

    def forward(self, x, t):
        self.x_in.tensor.copy_(x)
        self.t_in.tensor.copy_(t)
        draw_dropout_masks(self.fwd)
        self.fwd.run()
        return _tensor_of(self.out, (self.B, self.net.input_channel)).clone()

    def backward(self, d_out):
        self.d_out.tensor.copy_(d_out)
        self.bwd.run()
        grads = self.sink.collect()
        return [grads.get(id(p)) for p in self.params]


class _MLPFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, trainer: MLPTrainer, x, t, *params):
        ctx.trainer = trainer
        ctx.gen = trainer._stamp()
        with torch.no_grad():
            return trainer.forward(x, t)

    @staticmethod
    def backward(ctx, d_out):
        ctx.trainer._claim(ctx.gen, "MLPSkipNet")
        with torch.no_grad():
            pg = ctx.trainer.backward(d_out.contiguous())
        return (None, None, None, *pg)


def mlp_train_forward(net, x, t):
    B = x.shape[0]
    cache = net.__dict__.setdefault("_train_cache", {})
    amp = autocast_active() and mlp_amp_supported(net)
    key = (B, net.training, amp)
    tr = cache.get(key)
    if tr is None or tr.fwd.stale() or tr.bwd.stale():
        tr = MLPTrainer(net, B, amp)
        cache[key] = tr
    return _MLPFn.apply(tr, x, t, *tr.params)
