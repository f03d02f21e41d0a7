"""Semantic encoders x0 -> z (reference: model/representation_learning/encoder/*.py).

Five near-identical stride-2 conv stacks; CelebA64 is the 4-stage / 64 px variant (celeba64.py:10-37), the
others the 5-stage / 128 px variant (ffhq.py:10-41 == celebahq / bedroom / horse).  The nn.Sequential index
numbering of the reference (``encoder.{idx}``) is reproduced with explicit slots.
"""
from __future__ import annotations

from typing import List

import torch
import torch.nn as nn

from ....engine import Plan, RESAMPLE_NONE
from ...module import AttentionBlock, PlannedModule, Slots, Src, normalization


class ConvStackEncoder(PlannedModule):
    widths: List[int] = []
    attn_after = 0      # index into widths after which the AttentionBlock sits
    image_size = 0

    def __init__(self, **kwargs):
        super().__init__()
        self.latent_dim = kwargs["latent_dim"]
        w = self.widths
        slots = {0: nn.Conv2d(3, w[0], (3, 3), (2, 2), 1)}
        self._order = [("conv", 0)]
        idx, cin = 1, w[0]
        for j in range(1, len(w)):
            slots[idx] = normalization(cin)
            slots[idx + 2] = nn.Conv2d(cin, w[j], (3, 3), (2, 2), 1)
            self._order += [("gn", idx), ("conv", idx + 2)]
            idx += 3
            cin = w[j]
            if j == self.attn_after:
                slots[idx] = AttentionBlock(cin, 4, -1, False)
                self._order.append(("attn", idx))
                idx += 1
        slots[idx] = normalization(cin)
        self._order.append(("gn", idx))
        idx += 3  # GroupNorm, SiLU, View
        slots[idx] = nn.Linear(cin * 16, self.latent_dim)
        self._order.append(("linear", idx))
        self.encoder = Slots(slots)

    def _build(self, P: Plan, B: int, H: int, W: int):
        """The forward-only plan.  "fp32": every conv and the Linear on the CUDA cores.  "bf16" / "bf16x3": the stride-2 convs
        after the stem on the tensor cores (conv_tc2 through parity views) on the bf16 / split-operand GroupNorm-SiLU output,
        writing the stream dtype and the next GroupNorm's statistics; the final Linear as a bf16 / split-operand GEMM.  The
        stem computes in fp32 on the CUDA cores either way: the stride-2 stem kernel writing the bf16 stream and its statistics
        in "bf16", the fp32 conv in "bf16x3"."""
        x_in = P.new((B, 3, H, W), torch.float32, "x_nchw")
        x_in.keep = True
        h = None
        C = 3
        pending_ab = None  # (ab) of a GN whose SiLU output feeds the next conv
        z = None
        for kind, idx in self._order:
            m = self.encoder[idx]
            if kind == "conv":
                Co = m.weight.shape[0]
                Ho, Wo = H // 2, W // 2
                if h is None:
                    h = self._emit_stem(P, m, x_in, B, H, W)
                else:
                    tc = P.can_conv_s2(H, W, C, Co)
                    act, _ = P.gn_apply(h.b1, C, None, 0, pending_ab, silu=True, resample=RESAMPLE_NONE, B=B, H=H, W=W,
                                        act_dtype=torch.bfloat16 if tc else torch.float32)
                    out = P.new((B, Ho, Wo, Co), P.stream_dtype if tc else torch.float32, "enc_h")
                    st = P.conv(act, m.weight, m.bias, out, B=B, H=H, W=W, Cin=C, Cout=Co, k=3, stride=2, pad=1,
                                want_stats=tc)
                    h = Src(out, Co, B, Ho, Wo, s1=st)
                C, H, W = Co, Ho, Wo
            elif kind == "gn":
                pending_ab = P.gn_coef(h.b1, C, None, 0, m.weight, m.bias, B=B, HW=H * W, stats1=h.s1)
            elif kind == "attn":
                h = m.emit(P, h)
            else:  # final GN+SiLU, View(-1, C*4*4) in NCHW order, Linear
                z = P.new((B, self.latent_dim), torch.float32, "z")
                z.keep = True
                self._emit_linear(P, m, h, pending_ab, z, B, H, W, C)
        return x_in, z

    def _emit_stem(self, P: Plan, m: nn.Conv2d, x_in, B: int, H: int, W: int) -> Src:
        Co = m.weight.shape[0]
        Ho, Wo = H // 2, W // 2
        if P.stream_bf16 and Co % 8 == 0 and Co <= 256 and W % 8 == 0 and P.stem_det_fits(3, Co):
            # bf16 stream from the first layer: the stride-2 stem writes bf16 NHWC and the first GroupNorm's statistics
            wt = m.weight
            wp = P.pack((id(wt), "stem"), [wt], lambda: wt.detach().reshape(Co, 3, 9).permute(2, 1, 0).float())   # [9][Cin][Cout]
            out = P.new((B, Ho, Wo, Co), torch.bfloat16, "enc_stem")
            st = P.stem_conv_bf16(x_in, wp, m.bias, out, B=B, H=H, W=W, Cin=3, Cout=Co, stride=2,
                                  flops=2.0 * B * Ho * Wo * Co * 3 * 9)
            return Src(out, Co, B, Ho, Wo, s1=st)
        out = P.new((B, Ho, Wo, Co), torch.float32, "enc_h")
        P.conv(x_in, m.weight, m.bias, out, B=B, H=H, W=W, Cin=3, Cout=Co, k=3, stride=2, pad=1, in_nchw=True)
        return Src(out, Co, B, Ho, Wo)

    def _emit_linear(self, P: Plan, m: nn.Linear, h: Src, pending_ab, z, B: int, H: int, W: int, C: int) -> None:
        # the reference flattens NCHW (c, y, x); our activation is NHWC (y, x, c): permute the weight instead
        wt = m.weight
        HW, D = H * W, self.latent_dim
        tc = P.tc and D % 64 == 0 and (HW * C) % 64 == 0
        act, _ = P.gn_apply(h.b1, C, None, 0, pending_ab, silu=True, resample=RESAMPLE_NONE, B=B, H=H, W=W,
                            act_dtype=torch.bfloat16 if tc else torch.float32)
        if not tc:
            wp = P.pack((id(wt), "enc_fc"), [wt],
                        lambda: wt.detach().reshape(-1, C, HW).permute(2, 1, 0).reshape(HW * C, -1).float())
            P.linear_packed(act, wp, P.param(m.bias), z, B=B, Cin=HW * C, Cout=D)
            return
        if P.x3:
            # per pixel [W_hi | W_hi | W_lo] against the activation's [a_hi | a_lo | a_hi] blocks: K = 3 HW C
            def pack_x3():
                w = wt.detach().reshape(D, C, HW).permute(0, 2, 1).float()          # [D][HW][C]
                hi = w.to(torch.bfloat16)
                lo = (w - hi.float()).to(torch.bfloat16)
                return torch.cat([hi, hi, lo], dim=2).reshape(D, 3 * HW * C)
            wp = P.pack((id(wt), "enc_fc_x3"), [wt], pack_x3)
            K = 3 * HW * C
        else:
            wp = P.pack((id(wt), "enc_fc_tc"), [wt],
                        lambda: wt.detach().reshape(D, C, HW).permute(0, 2, 1).reshape(D, HW * C).to(torch.bfloat16))
            K = HW * C
        P.linear_tc(act, wp, P.param(m.bias), B=B, Cin=K, Cout=D, out=z, flops=2.0 * B * HW * C * D)

    def forward(self, x):
        """x [N,3,S,S] fp32 -> z [N, latent_dim]."""
        B, C, H, W = x.shape
        assert C == 3
        if (H, W) != (self.image_size, self.image_size):
            raise ValueError(f"{type(self).__name__} is hard-wired to {self.image_size}x{self.image_size} inputs "
                             f"(View(-1, C*4*4) in the reference), got {H}x{W}")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            from ....train import encoder_train_forward
            return encoder_train_forward(self, x.contiguous())
        plan, (x_in, z) = self._get_plan(("enc", B, H, W), lambda P: self._build(P, B, H, W))
        x_in.tensor.copy_(x)
        plan.run()
        return z.tensor.clone()


class Encoder64(ConvStackEncoder):
    widths = [64, 128, 128, 128]
    attn_after = 1
    image_size = 64


class Encoder128(ConvStackEncoder):
    widths = [64, 128, 256, 256, 256]
    attn_after = 2
    image_size = 128
