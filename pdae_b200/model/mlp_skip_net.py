"""Latent DPM: MLP with input skip-concat, time-conditioned scale, LayerNorm, SiLU
(reference surface: model/mlp_skip_net.py:6-141), as one native plan.

Per layer i: h = Linear([h | x] if i >= 1 else h); if conditioned: h = h * (1 + Linear(SiLU(cond))); LayerNorm;
SiLU; the last layer is Linear only.  The concat is free: every layer writes its output into the left columns of
a [B, width + in] buffer whose right columns hold x.  In the "bf16" / "bf16x3" modes the Linears run on the tensor cores on
split operands (_build_tc); "fp32" runs them on the CUDA cores.
"""
from __future__ import annotations

import ctypes

import torch
import torch.nn as nn

from ..engine import Plan, _STREAM, get_default_precision, split3_weights
from .module import PlannedModule, Slots, timestep_freqs


class MLPLNAct(nn.Module):
    """Parameter holder with the reference's keys: linear, linear_emb (+ alias cond_layers.1), norm."""

    def __init__(self, in_channels, out_channels, norm, use_cond, activation, cond_channels, dropout):
        super().__init__()
        self.activation = activation
        self.use_cond = use_cond
        self.linear = nn.Linear(in_channels, out_channels)
        self.act = nn.SiLU() if activation == "silu" else nn.Identity()
        if use_cond:
            self.linear_emb = nn.Linear(cond_channels, out_channels)
            self.cond_layers = nn.Sequential(self.act, self.linear_emb)
        self.norm = nn.LayerNorm(out_channels) if norm else nn.Identity()
        self.dropout = nn.Dropout(p=dropout) if dropout > 0 else nn.Identity()
        if activation == "silu":  # reference init_weights(): kaiming-normal on every Linear of a SiLU layer
            for m in self.modules():
                if isinstance(m, nn.Linear):
                    nn.init.kaiming_normal_(m.weight, a=0, nonlinearity="relu")


class MLPSkipNet(PlannedModule):
    def __init__(self, input_channel, model_channel, num_layers, time_emb_channel, use_norm, dropout, **kwargs):
        super().__init__()
        self.input_channel = input_channel
        self.model_channel = model_channel
        self.skip_layers = list(range(1, num_layers))
        self.time_emb_channel = time_emb_channel
        self.time_embed = Slots({0: nn.Linear(time_emb_channel, input_channel), 2: nn.Linear(input_channel, input_channel)})
        self.layers = nn.ModuleList()
        for i in range(num_layers):
            last = i == num_layers - 1
            a = input_channel if i == 0 else model_channel + input_channel
            b = input_channel if last else model_channel
            self.layers.append(MLPLNAct(a, b, norm=use_norm and not last, activation="none" if last else "silu",
                                        cond_channels=input_channel, use_cond=not last, dropout=0 if last else dropout))

    def _tc_plan(self, precision: str) -> bool:
        """Does a forward-only plan in `precision` run the split-operand tensor-core plan (_build_tc)?  Both tensor-core modes
        do when every Linear but time_embed has Cin and Cout multiples of 64 (the AMP trainer's rule); other nets keep the
        CUDA-core plan in every mode."""
        from ..train import mlp_amp_supported
        return precision in ("bf16", "bf16x3") and mlp_amp_supported(self)

    def _build(self, P: Plan, B: int, one_t: bool = False):
        if self._tc_plan(P.precision):
            return self._build_tc(P, B, one_t)
        dev = self._device()
        D, Wd, Te = self.input_channel, self.model_channel, self.time_emb_channel
        x_in = P.new((B, D), torch.float32, "z_t")
        t_in = P.new((B,), torch.int64, "t")
        x_in.keep = t_in.keep = True
        temb = P.new((B, Te), torch.float32, "temb")
        P.call("timestep_embedding", t_in, B, Te, P.fixed(timestep_freqs(Te, dev)), temb, _STREAM)
        c0 = P.new((B, D), torch.float32, "cond_h")
        P.linear(temb, self.time_embed[0].weight, self.time_embed[0].bias, c0, B=B, Cin=Te, Cout=D)
        cond = P.new((B, D), torch.float32, "cond")
        P.linear(c0, self.time_embed[2].weight, self.time_embed[2].bias, cond, B=B, Cin=D, Cout=D, a_silu=True)
        cat = [P.new((B, Wd + D), torch.float32, "cat0"), P.new((B, Wd + D), torch.float32, "cat1")]
        for c in cat:
            P.call("copy_cols", x_in, c, Wd + D, Wd, B, D, _STREAM)
        cur, cin = x_in, D
        out = None
        n = len(self.layers)
        for i, layer in enumerate(self.layers):
            if layer.training and isinstance(layer.dropout, nn.Dropout):
                raise NotImplementedError("pdae_b200: MLPSkipNet dropout is only active on the training path (grad enabled); "
                                          "call .eval() for sampling")
            last = i == n - 1
            co = layer.linear.weight.shape[0]
            h = P.new((B, co), torch.float32, "mlp_h")
            if last:
                h.keep = True
            P.linear(cur, layer.linear.weight, layer.linear.bias, h, B=B, Cin=cin, Cout=co)
            if last:
                out = h
                break
            cnd = P.new((B, co), torch.float32, "mlp_cond")
            P.linear(cond, layer.linear_emb.weight, layer.linear_emb.bias, cnd, B=B, Cin=D, Cout=co, a_silu=True)
            dst = cat[i % 2]
            ln = layer.norm if isinstance(layer.norm, nn.LayerNorm) else None
            P.call("mlp_mod_ln_act", h, cnd, P.param(ln.weight) if ln else None, P.param(ln.bias) if ln else None,
                   ctypes.c_float(ln.eps if ln else 1e-5), 1, dst, Wd + D, B, co, _STREAM)
            cur, cin = dst, Wd + D
        return x_in, t_in, out

    def _build_tc(self, P: Plan, B: int, one_t: bool):
        """The "bf16" / "bf16x3" plan: fp32-grade Linears on the tensor cores.  Every Linear but time_embed multiplies split
        operands, [a_hi | a_lo | a_hi] (K = 3 Cin) against [W_hi | W_hi | W_lo], with fp32 accumulation and output, split-K where
        its output tiles alone would leave SMs idle (Plan.linear_tc).  The layers' linear_emb, which all read SiLU(cond), are
        one bank GEMM over their concatenated weights, as in the AMP trainer; each layer's modulate / LayerNorm / SiLU reads its
        column block of the bank and writes the next Linear's split operand into the left columns of a split concat buffer
        whose right columns hold the split of z_t.  time_embed (Te -> D, SiLU, D -> D) stays fp32 on the CUDA cores.
        one_t: every row has t[0] (a sampling loop): the time embedding, time_embed and the bank run for that one row."""
        dev = self._device()
        D, Wd, Te = self.input_channel, self.model_channel, self.time_emb_channel
        bf16 = torch.bfloat16
        f32 = ctypes.c_float
        x_in = P.new((B, D), torch.float32, "z_t")
        t_in = P.new((B,), torch.int64, "t")
        x_in.keep = t_in.keep = True
        Bc = 1 if one_t else B
        temb = P.new((Bc, Te), torch.float32, "temb")
        P.call("timestep_embedding", t_in, Bc, Te, P.fixed(timestep_freqs(Te, dev)), temb, _STREAM)
        c0 = P.new((Bc, D), torch.float32, "cond_h")
        P.linear(temb, self.time_embed[0].weight, self.time_embed[0].bias, c0, B=Bc, Cin=Te, Cout=D)
        cond = P.new((Bc, D), torch.float32, "cond")
        P.linear(c0, self.time_embed[2].weight, self.time_embed[2].bias, cond, B=Bc, Cin=D, Cout=D, a_silu=True)
        scond = P.new((Bc, 3 * D), bf16, "silu_cond_x3")     # split SiLU(cond): the operand of the bank GEMM
        P.call("mlp_mod_ln_act_split3", cond, None, 0, None, None, f32(1e-5), 1, scond, D, 0, Bc, D, _STREAM)
        emb_layers = [layer for layer in self.layers if layer.use_cond]
        ws, bs = [l.linear_emb.weight for l in emb_layers], [l.linear_emb.bias for l in emb_layers]
        offsets = [0]
        for w in ws:
            offsets.append(offsets[-1] + w.shape[0])
        total = offsets[-1]
        for p in ws + bs:
            P.params.append((p, p.data_ptr()))
        wbank = P.pack(("mlp_bank_x3", id(ws[0])), ws,
                       lambda: split3_weights(torch.cat([w.detach() for w in ws], 0).reshape(total, D, 1))[0])
        bbank = P.pack(("mlp_bank_bias", id(bs[0])), bs, lambda: torch.cat([b.detach() for b in bs]).float())
        bank = P.linear_tc(scond, wbank, bbank, B=Bc, Cin=3 * D, Cout=total, name="mlp_bank", flops=2.0 * Bc * D * total)
        x3 = P.new((B, 3 * D), bf16, "z_t_x3")
        P.call("copy_cols_split3", x_in, x3, D, 0, B, D, _STREAM)
        cat = [P.new((B, 3 * (Wd + D)), bf16, "cat0_x3"), P.new((B, 3 * (Wd + D)), bf16, "cat1_x3")]
        for c in cat:
            P.call("copy_cols_split3", x_in, c, Wd + D, Wd, B, D, _STREAM)
        cur, cin = x3, D
        out = None
        n = len(self.layers)
        for i, layer in enumerate(self.layers):
            if layer.training and isinstance(layer.dropout, nn.Dropout):
                raise NotImplementedError("pdae_b200: MLPSkipNet dropout is only active on the training path (grad enabled); "
                                          "call .eval() for sampling")
            last = i == n - 1
            w = layer.linear.weight
            co = w.shape[0]
            wp = P.pack((id(w), "tc_x3"), [w], lambda w=w, co=co, cin=cin: split3_weights(w.detach().reshape(co, cin, 1))[0])
            if last:
                out = P.new((B, co), torch.float32, "mlp_h")
                out.keep = True
                P.linear_tc(cur, wp, P.param(layer.linear.bias), B=B, Cin=3 * cin, Cout=co, out=out, flops=2.0 * B * cin * co)
                break
            h = P.linear_tc(cur, wp, P.param(layer.linear.bias), B=B, Cin=3 * cin, Cout=co, name="mlp_h",
                            flops=2.0 * B * cin * co)
            dst = cat[i % 2]
            ln = layer.norm if isinstance(layer.norm, nn.LayerNorm) else None
            P.call("mlp_mod_ln_act_split3", h, bank.at(offsets[emb_layers.index(layer)]), 0 if one_t else total,
                   P.param(ln.weight) if ln else None, P.param(ln.bias) if ln else None, f32(ln.eps if ln else 1e-5), 1, dst,
                   Wd + D, 0, B, co, _STREAM)
            cur, cin = dst, Wd + D
        return x_in, t_in, out

    def plan_for(self, B: int, one_t: bool = False):
        """(plan, (x_in, t_in, eps)) -- static buffers a sampling loop can drive directly.  one_t: the plan of a batch whose
        rows share t[0] (the latent DDIM loop); in the tensor-core modes it runs the time embedding, time_embed and the
        linear_emb bank for one row, in "fp32" (and for nets kept on the CUDA cores) it is the per-row plan."""
        prec = self.precision or get_default_precision()
        if one_t and self._tc_plan(prec):
            return self._get_plan(("mlp_one_t", B, self.training), lambda P: self._build(P, B, one_t=True))
        return self._get_plan(("mlp", B, self.training), lambda P: self._build(P, B))

    def forward(self, x, t, condition=None):
        """x = z_t [N, input_channel], t int64 [N] -> predicted noise [N, input_channel]."""
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            # latent DPM training step (diffusion/gaussian_diffusion.py:373-398): hand-written backward for every parameter
            if x.requires_grad:
                raise NotImplementedError("pdae_b200: gradients w.r.t. z_t are not provided (the reference detaches z_0)")
            from ..train import mlp_train_forward
            return mlp_train_forward(self, x.contiguous(), t)
        self._check_no_grad(x)
        B = x.shape[0]
        plan, (x_in, t_in, out) = self.plan_for(B)
        x_in.tensor.copy_(x)
        t_in.tensor.copy_(t)
        plan.run()
        return out.tensor.clone()
