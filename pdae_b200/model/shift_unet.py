"""ShiftUNet: frozen epsilon-UNet + trainable z-conditioned "shift" decoder half
(reference surface: model/shift_unet.py:29-310), executed as one native plan per step.

forward(x, time, condition=z) -> (epsilon, shift).  Both decoder halves consume the same skip tensors of the
shared (frozen) encoder half; skip concatenations are never materialised (virtual two-source reads).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from ..engine import Plan
from .module import PlannedModule, Slots, TimestepSequential, conv_nd, linear
from .unet import EmbBank, emit_head, emit_stem, emit_time_embed, level_plan, make_head, make_middle, make_stage, res_blocks_of


class ShiftUNet(PlannedModule):
    def __init__(self, input_channel, base_channel, channel_multiplier, num_residual_blocks_of_a_block,
                 attention_resolutions, num_heads, head_channel, use_new_attention_order, dropout, latent_dim, dims=2,
                 learn_sigma=False, **kwargs):
        super().__init__()
        self.base_channel = base_channel
        self.input_channel = input_channel
        self.latent_dim = latent_dim
        self.output_channel = input_channel * 2 if learn_sigma else input_channel
        E = self.time_embed_dim = base_channel * 4
        topo = level_plan(base_channel, channel_multiplier, num_residual_blocks_of_a_block, attention_resolutions)
        attn_kw = dict(num_heads=num_heads, num_head_channels=head_channel, use_new_attention_order=use_new_attention_order)

        self.time_embed = Slots({0: linear(base_channel, E), 2: linear(E, E)})  # frozen (pre-trained DPM)
        self.label_emb = nn.Linear(latent_dim, E)                               # trainable: z -> shift embedding
        self.input_blocks = nn.ModuleList([TimestepSequential(conv_nd(dims, input_channel, topo["stem"], 3, padding=1))])
        for layers in topo["down"]:
            self.input_blocks.append(make_stage(layers, E, dropout, dims, attn_kw, False))
        self.middle_block = make_middle(topo["mid"], E, dropout, dims, attn_kw, False)
        self.shift_middle_block = make_middle(topo["mid"], E, dropout, dims, attn_kw, True)
        self.output_blocks = nn.ModuleList([make_stage(l, E, dropout, dims, attn_kw, False) for l in topo["up"]])
        self.shift_output_blocks = nn.ModuleList([make_stage(l, E, dropout, dims, attn_kw, True) for l in topo["up"]])
        self.out = make_head(topo["final"], topo["stem"], self.output_channel, dims)
        self.shift_out = make_head(topo["final"], topo["stem"], input_channel, dims)
        self.freeze()

    # ---- reference mode switches (model/shift_unet.py:287-310) --------------------------------------
    def _shift_parts(self):
        return (self.label_emb, self.shift_middle_block, self.shift_output_blocks, self.shift_out)

    def _frozen_parts(self):
        return (self.time_embed, self.input_blocks, self.middle_block, self.output_blocks, self.out)

    def set_train_mode(self):
        for m in self._shift_parts():
            m.train()

    def set_eval_mode(self):
        for m in self._shift_parts():
            m.eval()

    def freeze(self):
        for m in self._frozen_parts():
            m.eval()
            m.requires_grad_(requires_grad=False)

    # ---- plan ---------------------------------------------------------------------------------------
    def _build(self, P: Plan, B: int, H: int, W: int, with_shift: bool = True, interp: bool = False):
        """with_shift=False records only the frozen epsilon half (== the plain UNet): the plan a sampling loop replays on
        its `use_shift=False` tail steps (ddim.py:119, stop_percent > 0), skipping ~45 % of the FLOPs.
        interp=True: the trajectory-interpolation plan (ddim.py:149-174) -- two z inputs, the frozen half and the epsilon
        head once, one shift half per z on the same skip tensors; the second shift head is the plan's last op."""
        dev = self._device()
        E, base = self.time_embed_dim, self.base_channel
        x_in = P.new((B, self.input_channel, H, W), torch.float32, "x_nchw")
        t_in = P.new((B,), torch.int64, "t")
        z_ins = [P.new((B, self.latent_dim), torch.float32, n) for n in (("z", "z2") if interp else ("z",))]
        for b in (x_in, t_in, *z_ins):
            b.keep = True
        shift_blocks = res_blocks_of(self.shift_middle_block, self.shift_output_blocks) if with_shift else []
        banks_z = []
        if with_shift:
            # z is constant over a sampling loop: label_emb(z) and every emb_z_layers Linear are step-invariant
            # (SURVEY.md §8(f) row 2) -- recorded as the plan's prologue, run once per loop instead of once per step
            with P.prologue():
                for z_in in z_ins:
                    shift_emb = P.new((B, E), torch.float32, "shift_emb")
                    shift_emb.keep = True
                    P.linear(z_in, self.label_emb.weight, self.label_emb.bias, shift_emb, B=B, Cin=self.latent_dim, Cout=E)
                    bank_z = EmbBank(P, shift_blocks, "z", shift_emb, B, E, "shift_z")
                    bank_z.out.keep = True
                    banks_z.append(bank_z)
        emb = emit_time_embed(P, self.time_embed, t_in, B, base, E, dev)
        bank_t = EmbBank(P, res_blocks_of(self.input_blocks, self.middle_block, self.output_blocks) + shift_blocks, "t",
                         emb, B, E, "shift_t" if with_shift else "eps_t")

        h = emit_stem(P, self.input_blocks[0][0], x_in, B, H, W, self.input_channel)
        hs = [h]
        for stage in list(self.input_blocks)[1:]:
            h = stage.emit(P, h, bank_t)
            hs.append(h)
        eps_h = self.middle_block.emit(P, h, bank_t)
        shift_hs = [self.shift_middle_block.emit(P, h, bank_t, bank_z) for bank_z in banks_z]
        for stage, shift_stage in zip(self.output_blocks, self.shift_output_blocks):
            skip = hs.pop()
            eps_h = stage.emit(P, eps_h.cat(skip), bank_t)
            shift_hs = [shift_stage.emit(P, sh.cat(skip), bank_t, bank_z) for sh, bank_z in zip(shift_hs, banks_z)]
        eps = P.new((B, self.output_channel, H, W), torch.float32, "eps_nchw")
        eps.keep = True
        emit_head(P, self.out, eps_h, eps, fuse_key=None if with_shift else "eps")
        grads = []
        for k, shift_h in enumerate(shift_hs):
            grad = P.new((B, self.input_channel, H, W), torch.float32, "shift_nchw")
            grad.keep = True
            last = k == len(shift_hs) - 1   # the step's LAST op: may carry the fused sampling update
            emit_head(P, self.shift_out, shift_h, grad, fuse_key="grad" if last else None)
            grads.append(grad)
        if interp:
            return x_in, t_in, z_ins[0], z_ins[1], eps, grads[0], grads[1]
        return x_in, t_in, z_ins[0], eps, grads[0] if grads else None

    def plan_for(self, B: int, H: int, W: int, with_shift: bool = True):
        """(plan, (x_in, t_in, z_in, eps, grad)) -- static buffers a sampling loop can drive directly.
        with_shift=False: the epsilon-only plan (grad is None, z_in unused)."""
        return self._get_plan(("shiftunet" if with_shift else "shiftunet_eps", B, H, W, self.training),
                              lambda P: self._build(P, B, H, W, with_shift))

    def plan_for_interp(self, B: int, H: int, W: int):
        """(plan, (x_in, t_in, z1_in, z2_in, eps, g1, g2)) -- the trajectory-interpolation plan (see _build)."""
        return self._get_plan(("shiftunet_interp", B, H, W, self.training),
                              lambda P: self._build(P, B, H, W, interp=True))

    def forward(self, x, time, condition):
        """x [N,3,H,W], time int64 [N], condition = z [N, latent_dim] -> (epsilon, shift), both NCHW fp32."""
        if torch.is_grad_enabled() and (condition.requires_grad or
                                        any(p.requires_grad for m in self._shift_parts() for p in m.parameters())):
            # training step (gaussian_diffusion.py:234-255): hand-written backward behind a torch.autograd.Function
            if x.requires_grad:
                raise NotImplementedError("pdae_b200: gradients w.r.t. x_t are not provided (the reference never needs them)")
            from ..train import shiftunet_train_forward
            return shiftunet_train_forward(self, x.contiguous(), time, condition)
        B, C, H, W = x.shape
        assert C == self.input_channel
        plan, (x_in, t_in, z_in, eps, grad) = self.plan_for(B, H, W)
        x_in.tensor.copy_(x)
        t_in.tensor.copy_(time)
        z_in.tensor.copy_(condition)
        plan.run()
        return eps.tensor.clone(), grad.tensor.clone()
