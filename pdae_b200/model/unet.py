"""UNet (epsilon-prediction DPM) behind the reference's surface (model/unet.py:30-202), run as one native plan.

Constructor keywords, attribute names (``time_embed``, ``label_emb``, ``input_blocks``, ``middle_block``,
``output_blocks``, ``out``) and ``state_dict`` keys/shapes match the reference, so its checkpoints load with
``load_state_dict`` and its trainers/samplers can address sub-modules unchanged.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch
import torch.nn as nn

from ..engine import Buf, Plan, _STREAM
from .module import (AttentionBlock, PlannedModule, ResBlock, ResBlockShift, Slots, Src, TimestepSequential, conv_nd,
                     linear, normalization, timestep_freqs, zero_module)


def level_plan(base_channel: int, channel_multiplier, num_res: int, attention_resolutions) -> dict:
    """Channel/attention bookkeeping of the UNet topology (model/unet.py:60-169), as data.

    Returns {'stem': ch, 'down': [...], 'mid': ch, 'up': [...]} where each down/up entry is a list of layer
    descriptors ('res', cin, cout, mode) / ('attn', ch); mode in {'', 'up', 'down'}."""
    widths = [int(m * base_channel) for m in channel_multiplier]
    attn = set(attention_resolutions)
    ch = widths[0]
    skip_ch = [ch]
    down: List[list] = []
    ds = 1
    for lvl, w in enumerate(widths):
        for _ in range(num_res):
            blk = [("res", ch, w, "")]
            ch = w
            if ds in attn:
                blk.append(("attn", ch))
            down.append(blk)
            skip_ch.append(ch)
        if lvl != len(widths) - 1:
            down.append([("res", ch, ch, "down")])
            skip_ch.append(ch)
            ds *= 2
    mid = ch
    up: List[list] = []
    for lvl in reversed(range(len(widths))):
        w = widths[lvl]
        for i in range(num_res + 1):
            blk = [("res", ch + skip_ch.pop(), w, "")]
            ch = w
            if ds in attn:
                blk.append(("attn", ch))
            if lvl and i == num_res:
                blk.append(("res", ch, ch, "up"))
                ds //= 2
            up.append(blk)
    return {"stem": widths[0], "down": down, "mid": mid, "up": up, "final": ch}


def make_stage(layers, emb_dim: int, dropout: float, dims: int, attn_kw: dict, shift: bool) -> TimestepSequential:
    mods = []
    for d in layers:
        if d[0] == "res":
            cls = ResBlockShift if shift else ResBlock
            mods.append(cls(d[1], emb_dim, dropout, out_channels=d[2], dims=dims, up=d[3] == "up", down=d[3] == "down"))
        else:
            mods.append(AttentionBlock(d[1], **attn_kw))
    return TimestepSequential(*mods)


def make_middle(ch: int, emb_dim: int, dropout: float, dims: int, attn_kw: dict, shift: bool) -> TimestepSequential:
    return make_stage([("res", ch, ch, ""), ("attn", ch), ("res", ch, ch, "")], emb_dim, dropout, dims, attn_kw, shift)


def make_head(ch: int, in_ch: int, out_ch: int, dims: int) -> Slots:
    """GN, SiLU, zero-init conv3x3 -> image channels (model/unet.py:171-175); keys '0' and '2'."""
    return Slots({0: normalization(ch), 2: zero_module(conv_nd(dims, in_ch, out_ch, 3, padding=1))})


class EmbBank:
    """All ``emb_layers`` (or ``emb_z_layers``) Linears of a network evaluated as ONE GEMM per step:
    the embedding is the same for every block, so their weights are concatenated along the output axis."""

    def __init__(self, P: Plan, blocks: List[nn.Module], which: str, emb: Buf, B: int, E: int, tag: str):
        lins = [(b.emb_layers[1] if which == "t" else b.emb_z_layers[1]) for b in blocks]
        self.offsets: Dict[int, int] = {}
        off = 0
        for b, l in zip(blocks, lins):
            self.offsets[id(b)] = off
            off += l.weight.shape[0]
        self.total = off
        ws = [l.weight for l in lins]
        bs = [l.bias for l in lins]
        wcat = P.pack((tag, "w"), ws, lambda: torch.cat([w.detach().t() for w in ws], dim=1).float())
        bcat = P.pack((tag, "b"), bs, lambda: torch.cat([b.detach() for b in bs]).float())
        self.out = P.new((B, self.total), torch.float32, "emb_bank_" + tag)
        P.linear_packed(emb, wcat, bcat, self.out, B=B, Cin=E, Cout=self.total, a_silu=True)

    def __call__(self, blk) -> Tuple[Buf, int, int]:
        return self.out, self.offsets[id(blk)], self.total


def emit_time_embed(P: Plan, time_embed: Slots, t: Buf, B: int, base: int, E: int, device) -> Buf:
    """time_embed(timestep_embedding(t, base)) (model/unet.py:188)."""
    freqs = P.fixed(timestep_freqs(base, device))
    temb = P.new((B, base), torch.float32, "temb")
    P.call("timestep_embedding", t, B, base, freqs, temb, _STREAM)
    h = P.new((B, E), torch.float32, "temb_h")
    P.linear(temb, time_embed[0].weight, time_embed[0].bias, h, B=B, Cin=base, Cout=E)
    emb = P.new((B, E), torch.float32, "emb")
    P.linear(h, time_embed[2].weight, time_embed[2].bias, emb, B=B, Cin=E, Cout=E, a_silu=True)
    return emb


def emit_stem(P: Plan, stem: nn.Module, x_in: Buf, B: int, H: int, W: int, Cin: int) -> Src:
    """First conv of the network on the NCHW image (model/unet.py:62-64).  With the bf16 residual stream it is ONE launch
    writing bf16 NHWC plus the per-channel sums the first GroupNorms need (the stem output is a skip tensor read by three
    of them); otherwise the generic CUDA-core conv (+ a statistics pass in fused-statistics mode)."""
    c0 = stem.weight.shape[0]
    if (P.fused_stats and P.stream_bf16 and Cin <= 4 and c0 % 8 == 0 and c0 <= 256 and stem.kernel_size[0] == 3
            and W % 4 == 0 and P.stem_det_fits(Cin, c0)):
        wt = stem.weight
        wp = P.pack((id(wt), "stem"), [wt], lambda: wt.detach().reshape(c0, Cin, 9).permute(2, 1, 0).float())   # [9][Cin][Cout]
        h0 = P.new((B, H, W, c0), torch.bfloat16, "stem")
        st0 = P.stem_conv_bf16(x_in, wp, stem.bias, h0, B=B, H=H, W=W, Cin=Cin, Cout=c0, stride=1,
                               flops=2.0 * B * H * W * c0 * Cin * 9)
        return Src(h0, c0, B, H, W, s1=st0)
    h0 = P.new((B, H, W, c0), torch.float32, "stem")
    P.conv(x_in, stem.weight, stem.bias, h0, B=B, H=H, W=W, Cin=Cin, Cout=c0, k=3, in_nchw=True)
    st0 = P.ch_stats(h0, c0, B=B, HW=H * W) if P.fused_stats else None
    return Src(P.to_stream(h0, c0, B=B, H=H, W=W), c0, B, H, W, s1=st0)


def emit_head(P: Plan, head: Slots, x: Src, out: Buf, tape=None, fuse_key=None) -> None:
    gn, conv = head[0], head[2]
    B, H, W, C = x.B, x.H, x.W, x.C
    ab = P.gn_coef(x.b1, C, None, 0, gn.weight, gn.bias, B=B, HW=H * W, stats1=x.s1)
    sums = P.last_sums
    act, _ = P.gn_apply(x.b1, C, None, 0, ab, silu=True, resample=0, B=B, H=H, W=W,
                        act_dtype=P.head_act_dtype(C, conv.weight.shape[0], H, W))
    P.head_conv(act, conv.weight, conv.bias, out, B=B, H=H, W=W, Cin=C, Cout=conv.weight.shape[0],
                fuse_key=fuse_key if tape is None else None)
    if tape is not None:
        tape.append(("head", head, dict(x=x, ab=ab, sums=sums, act=act)))


def res_blocks_of(*containers) -> List[nn.Module]:
    out = []
    for c in containers:
        for m in c.modules():
            if isinstance(m, (ResBlock, ResBlockShift)):
                out.append(m)
    return out


class UNet(PlannedModule):
    def __init__(self, input_channel, base_channel, channel_multiplier, num_residual_blocks_of_a_block,
                 attention_resolutions, num_heads, head_channel, use_new_attention_order, dropout, num_class=None, dims=2,
                 learn_sigma=False, **kwargs):
        super().__init__()
        self.num_class = num_class
        self.base_channel = base_channel
        self.input_channel = input_channel
        self.output_channel = input_channel * 2 if learn_sigma else input_channel
        E = self.time_embed_dim = base_channel * 4
        topo = level_plan(base_channel, channel_multiplier, num_residual_blocks_of_a_block, attention_resolutions)
        attn_kw = dict(num_heads=num_heads, num_head_channels=head_channel, use_new_attention_order=use_new_attention_order)

        self.time_embed = Slots({0: linear(base_channel, E), 2: linear(E, E)})
        if num_class is not None:
            self.label_emb = nn.Embedding(num_class, E)
        self.input_blocks = nn.ModuleList([TimestepSequential(conv_nd(dims, input_channel, topo["stem"], 3, padding=1))])
        for layers in topo["down"]:
            self.input_blocks.append(make_stage(layers, E, dropout, dims, attn_kw, False))
        self.middle_block = make_middle(topo["mid"], E, dropout, dims, attn_kw, False)
        self.output_blocks = nn.ModuleList([make_stage(layers, E, dropout, dims, attn_kw, False) for layers in topo["up"]])
        self.out = make_head(topo["final"], topo["stem"], self.output_channel, dims)

    def _build(self, P: Plan, B: int, H: int, W: int):
        dev = self._device()
        E, base = self.time_embed_dim, self.base_channel
        x_in = P.new((B, self.input_channel, H, W), torch.float32, "x_nchw")
        t_in = P.new((B,), torch.int64, "t")
        c_in = P.new((B,), torch.int64, "cond") if self.num_class is not None else None
        for b in (x_in, t_in, c_in):
            if b is not None:
                b.keep = True
        emb = emit_time_embed(P, self.time_embed, t_in, B, base, E, dev)
        if c_in is not None:
            P.call("embedding_add", emb, P.param(self.label_emb.weight), c_in, B, E, _STREAM)
        bank = EmbBank(P, res_blocks_of(self.input_blocks, self.middle_block, self.output_blocks), "t", emb, B, E, "unet_t")

        h = emit_stem(P, self.input_blocks[0][0], x_in, B, H, W, self.input_channel)
        hs = [h]
        for stage in list(self.input_blocks)[1:]:
            h = stage.emit(P, h, bank)
            hs.append(h)
        h = self.middle_block.emit(P, h, bank)
        for stage in self.output_blocks:
            h = stage.emit(P, h.cat(hs.pop()), bank)
        out = P.new((B, self.output_channel, H, W), torch.float32, "eps_nchw")
        out.keep = True
        emit_head(P, self.out, h, out, fuse_key="eps")
        return x_in, t_in, c_in, out

    def plan_for(self, B: int, H: int, W: int):
        """(plan, (x_in, t_in, c_in, eps)) -- static buffers a sampling loop can drive directly (c_in: class labels or None)."""
        return self._get_plan(("unet", B, H, W), lambda P: self._build(P, B, H, W))

    def forward(self, x, time, condition=None):
        """x [N,C,H,W] fp32, time int64 [N], condition int64 [N] if class-conditional -> [N,C(|2C),H,W]."""
        if self.num_class is not None:
            assert condition is not None
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            if x.requires_grad:
                raise NotImplementedError("pdae_b200: gradients w.r.t. x_t are not provided (the reference never needs them)")
            from ..train import unet_train_forward   # regular DPM training step (gaussian_diffusion.py:199-211)
            return unet_train_forward(self, x.contiguous(), time, condition)
        B, C, H, W = x.shape
        assert C == self.input_channel
        plan, (x_in, t_in, c_in, out) = self.plan_for(B, H, W)
        x_in.tensor.copy_(x)
        t_in.tensor.copy_(time)
        if c_in is not None:
            c_in.tensor.copy_(condition)
        plan.run()
        return out.tensor.clone()
