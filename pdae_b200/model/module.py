"""Building blocks with the reference's parameter names, executed by the native kernels.

Same class names, constructor arguments, attribute names and ``state_dict`` keys as the reference's
``model/module.py`` (ResBlock :205-297, ResBlockShift :299-384, AttentionBlock :387-428, Upsample/Downsample
:143-202, TimestepSequential :131-140, timestep_embedding :66-84) -- but the modules here only *hold*
parameters; ``forward`` records/replays a launch plan over libpdae_b200 (pdae_b200.engine).  There is no
PyTorch-op fallback: a forward on a CPU tensor, or without the built library, raises.

Layout: parameters stay nn-style fp32 (NCHW conv weights) so checkpoints, DDP, Adam and EMA code written
against the reference keep working; activations inside a plan are NHWC.
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, Optional, Tuple

import torch
import torch.nn as nn

from .. import _native
from ..engine import Buf, Plan, RESAMPLE_DOWN2, RESAMPLE_NONE, RESAMPLE_UP2, _STREAM, get_default_precision


# --------------------------------------------------------------------------------------------------
# parameter holders
# --------------------------------------------------------------------------------------------------
class Slots(nn.Module):
    """Children registered under explicit integer names -- reproduces the key numbering of the reference's
    nn.Sequential containers (whose parameter-free members such as SiLU/Dropout leave gaps)."""

    def __init__(self, members: Dict[int, nn.Module]):
        super().__init__()
        for i, m in members.items():
            self.add_module(str(i), m)

    def __getitem__(self, i: int) -> nn.Module:
        return self._modules[str(i)]

    def __iter__(self):
        return iter(self._modules.values())

    def __len__(self):
        return len(self._modules)


def conv_nd(dims, *args, **kwargs):
    if dims == 1:
        return nn.Conv1d(*args, **kwargs)
    if dims == 2:
        return nn.Conv2d(*args, **kwargs)
    raise ValueError(f"pdae_b200 supports dims in (1, 2), got {dims}")


def linear(*args, **kwargs):
    return nn.Linear(*args, **kwargs)


def normalization(channels):
    """GroupNorm(32, C) parameters (model/module.py:56-63)."""
    return nn.GroupNorm(32, channels)


def zero_module(module):
    for p in module.parameters():
        p.detach().zero_()
    return module


class View(nn.Module):
    def __init__(self, size):
        super().__init__()
        self.size = size


_FREQ_CACHE: Dict[Tuple[int, str], torch.Tensor] = {}


def timestep_freqs(dim: int, device, max_period: int = 10000) -> torch.Tensor:
    """exp(-ln(max_period) * i / half), evaluated on the host with the reference's fp32 op order
    (model/module.py:75-79) and cached on the device."""
    key = (dim, str(device), max_period)
    if key not in _FREQ_CACHE:
        half = dim // 2
        f = torch.exp(-math.log(max_period) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
        _FREQ_CACHE[key] = f.to(device)
    return _FREQ_CACHE[key]


def timestep_embedding(timesteps: torch.Tensor, dim: int, max_period: int = 10000) -> torch.Tensor:
    """Sinusoidal embedding [N, dim] (cos | sin | zero pad) computed by pdae_timestep_embedding."""
    if not timesteps.is_cuda:
        raise _native.NativeError("timestep_embedding: CUDA tensor required (no CPU fallback)")
    t = timesteps.to(torch.int64).contiguous()
    out = torch.empty(t.shape[0], dim, device=t.device, dtype=torch.float32)
    L = _native.lib()
    import ctypes
    rc = L.pdae_timestep_embedding(ctypes.c_void_p(t.data_ptr()), t.shape[0], dim,
                                   ctypes.c_void_p(timestep_freqs(dim, t.device, max_period).data_ptr()),
                                   ctypes.c_void_p(out.data_ptr()),
                                   ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream))
    _native.check(rc, "pdae_timestep_embedding")
    return out


# --------------------------------------------------------------------------------------------------
# plan plumbing shared by every module
# --------------------------------------------------------------------------------------------------
class Src:
    """An NHWC fp32 activation, possibly the virtual channel-concat of two tensors (skip connections are
    never materialised: unet.py:199-200 / shift_unet.py:276-281 ``torch.cat([h, hs.pop()], 1)``)."""
    __slots__ = ("b1", "C1", "b2", "C2", "B", "H", "W", "s1", "s2")

    def __init__(self, b1: Buf, C1: int, B: int, H: int, W: int, b2: Optional[Buf] = None, C2: int = 0,
                 s1: Optional[Buf] = None, s2: Optional[Buf] = None):
        self.b1, self.C1, self.b2, self.C2, self.B, self.H, self.W = b1, C1, b2, C2, B, H, W
        self.s1, self.s2 = s1, s2  # per-channel (sum, sum^2) buffers accumulated by the producing conv's epilogue

    @property
    def C(self) -> int:
        return self.C1 + self.C2

    def cat(self, other: "Src") -> "Src":
        assert self.b2 is None and other.b2 is None and (self.B, self.H, self.W) == (other.B, other.H, other.W)
        return Src(self.b1, self.C1, self.B, self.H, self.W, other.b1, other.C1, self.s1, other.s1)


class PlannedModule(nn.Module):
    """Caches one plan per (input signature, precision, train flag); re-records if parameters moved."""

    precision: Optional[str] = None  # None -> engine default

    def _plans(self) -> dict:
        d = self.__dict__.get("_plan_cache")
        if d is None:
            d = {}
            self.__dict__["_plan_cache"] = d
        return d

    def _get_plan(self, key, builder):
        prec = self.precision or get_default_precision()
        # torch.use_deterministic_algorithms: the deterministic plan (engine.py), cached beside the default one
        det = torch.are_deterministic_algorithms_enabled()
        key = (key, prec, det)
        plans = self._plans()
        ent = plans.get(key)
        if ent is None or ent[0].stale():
            plan = Plan(self._device(), prec, deterministic=det)
            io = builder(plan)
            plan.finalize()
            ent = (plan, io)
            plans[key] = ent
        return ent

    def invalidate_packed(self) -> None:
        """Force every cached plan of this module (and of its sub-modules) to re-derive its packed weight copies on the
        next run.  Needed only after an in-place weight update that bumps no autograd version counter outside a sampling
        loop (`p.data.mul_()`, raw-pointer writes): versioned updates (optimizers, load_state_dict, copy_) are detected,
        and every sampling loop re-packs once at its start anyway."""
        for m in self.modules():
            for cache_name in ("_plan_cache", "_train_cache"):
                for ent in (m.__dict__.get(cache_name) or {}).values():
                    plans = [ent[0]] if isinstance(ent, tuple) else [getattr(ent, "fwd", None), getattr(ent, "bwd", None), getattr(ent, "frozen", None)]
                    for pl in plans:
                        if pl is not None:
                            for pk in pl.packed:
                                pk.stamp = None

    def _device(self) -> torch.device:
        p = next(self.parameters())
        if not p.is_cuda:
            raise _native.NativeError(f"{type(self).__name__}: parameters are on {p.device}; pdae_b200 runs on CUDA "
                                      "(sm_90) only -- there is no CPU fallback")
        return p.device

    def __deepcopy__(self, memo):
        # plans hold raw device pointers: never copy them (copy.deepcopy(decoder) is how the trainers make EMA nets)
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        import copy
        for k, v in self.__dict__.items():
            if k in ("_plan_cache", "_train_cache"):   # (trainer plans own native handles too: a copy would double-free them)
                continue
            new.__dict__[k] = copy.deepcopy(v, memo)
        return new

    def _check_no_grad(self, *tensors):
        """Forward-only for now: refuse (loudly) to run where autograd would expect a graph."""
        if not torch.is_grad_enabled():
            return
        if any(t is not None and t.requires_grad for t in tensors) or any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("pdae_b200: backward kernels are not built yet -- run under torch.no_grad() / "
                                      "inference_mode() (forward/sampling path)")


# --------------------------------------------------------------------------------------------------
# blocks
# --------------------------------------------------------------------------------------------------
class TimestepBlock(nn.Module):
    pass


class TimestepContextBlock(nn.Module):
    pass


class Upsample(nn.Module):
    """Parameter-free marker (the reference only ever builds it with use_conv=False, module.py:248-252)."""

    def __init__(self, channels, use_conv, dims=2, out_channels=None):
        super().__init__()
        assert not use_conv, "pdae_b200: Upsample(use_conv=True) is never constructed by the reference models"
        self.channels, self.out_channels, self.use_conv, self.dims = channels, out_channels or channels, use_conv, dims


class Downsample(nn.Module):
    def __init__(self, channels, use_conv, dims=2, out_channels=None):
        super().__init__()
        assert not use_conv, "pdae_b200: Downsample(use_conv=True) is never constructed by the reference models"
        self.channels, self.out_channels, self.use_conv, self.dims = channels, out_channels or channels, use_conv, dims


class _ResBase(PlannedModule):
    has_z = False

    def __init__(self, channels, emb_channels, dropout, out_channels=None, use_conv=False, dims=2, up=False, down=False):
        super().__init__()
        assert dims == 2, "only dims=2 is exercised by the reference configs"
        self.channels = channels
        self.emb_channels = emb_channels
        self.dropout = dropout
        self.out_channels = out_channels or channels
        self.use_conv = use_conv
        self.up, self.down = up, down
        self.updown = up or down
        co = self.out_channels
        self.in_layers = Slots({0: normalization(channels), 2: conv_nd(dims, channels, co, 3, padding=1)})
        if up:
            self.h_upd, self.x_upd = Upsample(channels, False, dims), Upsample(channels, False, dims)
        elif down:
            self.h_upd, self.x_upd = Downsample(channels, False, dims), Downsample(channels, False, dims)
        else:
            self.h_upd = self.x_upd = nn.Identity()
        self.emb_layers = Slots({1: linear(emb_channels, 2 * co)})
        if self.has_z:
            self.emb_z_layers = Slots({1: linear(emb_channels, 2 * co)})
        self.out_layers = Slots({0: normalization(co), 3: zero_module(conv_nd(dims, co, co, 3, padding=1))})
        if co == channels:
            self.skip_connection = nn.Identity()
        else:
            self.skip_connection = conv_nd(dims, channels, co, 3 if use_conv else 1, padding=1 if use_conv else 0)

    # ---- plan emission --------------------------------------------------------------------------
    def emit(self, P: Plan, x: Src, emb: Tuple[Buf, int, int], embz: Optional[Tuple[Buf, int, int]] = None,
             tape: Optional[list] = None) -> Src:
        """emb / embz = (buffer, element offset of this block's [scale|shift] row slice, leading dim).
        tape (training plans): receives the buffers the backward pass needs."""
        drop = self.training and self.dropout > 0
        if drop and tape is None:
            raise NotImplementedError("pdae_b200: dropout is only active on the training path (grad enabled); "
                                      "call .eval() / set_eval_mode() for sampling")
        assert x.C == self.channels, f"expected {self.channels} channels, got {x.C}"
        B, H, W, C, Co = x.B, x.H, x.W, x.C, self.out_channels
        rs = RESAMPLE_UP2 if self.up else (RESAMPLE_DOWN2 if self.down else RESAMPLE_NONE)
        H2, W2 = (2 * H, 2 * W) if self.up else ((H // 2, W // 2) if self.down else (H, W))
        conv1, conv2 = self.in_layers[2], self.out_layers[3]
        gn1, gn2 = self.in_layers[0], self.out_layers[0]
        ident = isinstance(self.skip_connection, nn.Identity)

        ab1 = P.gn_coef(x.b1, x.C1, x.b2, x.C2, gn1.weight, gn1.bias, B=B, HW=H * W, stats1=x.s1, stats2=x.s2)
        sums1 = P.last_sums
        eb, eoff, eld = emb
        zb = zoff = zld = None
        if self.has_z:
            zb, zoff, zld = embz
        # ---- fused-prologue path (conv_tc3): GN-apply / AdaGN / SiLU (and the hi/lo split) happen inside the convs' operand
        # path; the activated tensors act1 / act2 and the concatenated raw input never exist in HBM ----
        srcs = [(x.b1, x.C1), (x.b2, x.C2)]
        fuse2 = tape is None and not drop and P.can_fuse_prologue([(None, Co)], Co, H2, W2) and \
            (ident or (self.skip_connection.kernel_size[0] == 1 and P.can_fuse_prologue(srcs, Co, H2, W2)))
        fuse1 = fuse2 and not self.updown and P.can_fuse_prologue(srcs, Co, H, W)
        if fuse2 and (fuse1 or self.updown) and (not ident or self.updown or x.b2 is None):
            sdt = torch.float32 if P.x3 else torch.bfloat16          # this mode's stream dtype == conv_tc3's source dtype
            raw = None
            if fuse1:
                h = P.new((B, H2, W2, Co), sdt, "res_h")
                hs = P.conv_fused(x.b1, x.C1, x.b2, x.C2, ab1, conv1.weight, conv1.bias, h, B=B, H=H2, W=W2, Cout=Co,
                                  want_stats=True)
            else:
                # up / down-sampling block: the resample (of both the activated h and the raw x, module.py:282-288) stays a
                # gn_apply pass; its conv1 runs on conv_tc2, conv2 below on conv_tc3
                act1, raw = P.gn_apply(x.b1, x.C1, x.b2, x.C2, ab1, silu=True, resample=rs, B=B, H=H, W=W,
                                       act_dtype=torch.bfloat16, raw_dtype=sdt)
                h = P.new((B, H2, W2, Co), sdt, "res_h")
                hs = P.conv(act1, conv1.weight, conv1.bias, h, B=B, H=H2, W=W2, Cin=C, Cout=Co, k=3, want_stats=True)
            ab2 = P.gn_coef(h, Co, None, 0, gn2.weight, gn2.bias, B=B, HW=H2 * W2, emb=eb.at(eoff), emb_ld=eld,
                            embz=zb.at(zoff) if zb is not None else None, embz_ld=zld or 0, stats1=hs)
            out = P.new((B, H2, W2, Co), sdt, "res_out")
            if ident:
                resid = raw if raw is not None else x.b1
                assert resid.dtype == sdt
                os_ = P.conv_fused(h, Co, None, 0, ab2, conv2.weight, conv2.bias, out, B=B, H=H2, W=W2, Cout=Co, residual=resid,
                                   want_stats=True)
            else:
                sk = self.skip_connection
                k1, S1, k2, S2 = (raw, C, None, 0) if raw is not None else (x.b1, x.C1, x.b2, x.C2)
                os_ = P.conv_fused(h, Co, None, 0, ab2, conv2.weight, conv2.bias, out, B=B, H=H2, W=W2, Cout=Co,
                                   skip=(k1, S1, k2, S2, sk.weight, sk.bias), want_stats=True)
            return Src(out, Co, B, H2, W2, s1=os_)

        tc1 = P.use_tc(C, Co, 3, 1, H2, W2)
        tc2 = P.use_tc(Co, Co, 3, 1, H2, W2)
        tcs = (not ident) and P.use_tc(C, Co, self.skip_connection.kernel_size[0], 1, H2, W2)
        # dtype of this block's output (the residual stream): bf16 only when every conv of the block is a tensor-core one
        out_dt = P.stream_dtype if (tc1 and tc2 and (ident or tcs)) else torch.float32
        # raw (un-normalised) copy of the possibly concatenated / resampled input for the skip path
        plain = not self.updown and x.b2 is None        # x.b1 itself is the skip-path input
        # a concatenated input whose 1x1 skip conv is folded into conv2 is read from its two source tensors directly
        # (two TMA maps): the concat is never materialised
        cat_skip = (not ident and not self.updown and x.b2 is not None and tcs and tc2
                    and self.skip_connection.kernel_size[0] == 1 and x.b1.dtype == torch.bfloat16
                    and x.b2.dtype == torch.bfloat16 and x.C1 % 64 == 0 and x.C2 % 64 == 0 and tape is None)
        raw_dtype = None
        if cat_skip:
            pass
        elif ident:
            if not (plain and x.b1.dtype == out_dt):
                raw_dtype = out_dt                       # identity residual must have the output's dtype
        else:
            want = torch.bfloat16 if tcs else torch.float32
            if not (plain and x.b1.dtype == want):
                raw_dtype = want
        act1, raw = P.gn_apply(x.b1, x.C1, x.b2, x.C2, ab1, silu=True, resample=rs, B=B, H=H, W=W,
                               act_dtype=torch.bfloat16 if tc1 else torch.float32, raw_dtype=raw_dtype)
        # h only feeds GroupNorm-2: on the tensor cores it is stored in bf16 and its statistics come from the epilogue
        h_bf16 = tc1 and P.fused_stats and not P.x3     # (the split-operand mode keeps every conv output in fp32)
        h = P.new((B, H2, W2, Co), torch.bfloat16 if h_bf16 else torch.float32, "res_h")
        hs = P.conv(act1, conv1.weight, conv1.bias, h, B=B, H=H2, W=W2, Cin=C, Cout=Co, k=3, want_stats=True)

        eb, eoff, eld = emb
        zb = zoff = zld = None
        if self.has_z:
            zb, zoff, zld = embz
        ab2 = P.gn_coef(h, Co, None, 0, gn2.weight, gn2.bias, B=B, HW=H2 * W2, emb=eb.at(eoff), emb_ld=eld,
                        embz=zb.at(zoff) if zb is not None else None, embz_ld=zld or 0, stats1=hs)
        sums2 = P.last_sums
        act2, _ = P.gn_apply(h, Co, None, 0, ab2, silu=True, resample=RESAMPLE_NONE, B=B, H=H2, W=W2,
                             act_dtype=torch.bfloat16 if tc2 else torch.float32)
        mask = None
        if drop:   # nn.Dropout(p) between SiLU and conv2 (module.py:259): 0/1 mask drawn by the trainer every step
            mask = P.new((B, H2, W2, Co), torch.float32, "drop_mask")
            mask.keep = True
            P.dropout_masks.append((self, mask, float(self.dropout)))
            P.call("mul_mask", act2, mask, ctypes.c_float(1.0 / (1.0 - self.dropout)), ctypes.c_int64(B * H2 * W2 * Co), _STREAM)
        out = P.new((B, H2, W2, Co), out_dt, "res_out")
        fused_skip = None
        if ident:
            resid = raw if raw is not None else x.b1
        else:
            sk = self.skip_connection
            sk_in = (x.b1, x.C1, x.b2, x.C2) if cat_skip else (raw if raw is not None else x.b1)
            if cat_skip or (tcs and tc2 and sk.kernel_size[0] == 1 and sk_in.dtype == torch.bfloat16):
                resid, fused_skip = None, (sk_in, sk.weight, sk.bias, C)   # folded into conv2 as extra K blocks
            else:
                resid = P.new((B, H2, W2, Co), out_dt, "res_skip")
                P.conv(sk_in, sk.weight, sk.bias, resid, B=B, H=H2, W=W2, Cin=C, Cout=Co, k=sk.kernel_size[0])
        os_ = P.conv(act2, conv2.weight, conv2.bias, out, B=B, H=H2, W=W2, Cin=Co, Cout=Co, k=3, residual=resid,
                     want_stats=True, skip=fused_skip)
        if tape is not None:
            tape.append(("res", self, dict(x=x, ab1=ab1, sums1=sums1, act1=act1, raw=raw, h=h, sums2=sums2, ab2=ab2, act2=act2,
                                           emb=emb, embz=embz, rs=rs, ident=ident, H2=H2, W2=W2, mask=mask)))
        return Src(out, Co, B, H2, W2, s1=os_)

    def emit_emb(self, P: Plan, emb: Buf, B: int, which: str = "t") -> Tuple[Buf, int, int]:
        """This block's own Linear(SiLU(emb)) -> [B, 2*Cout] (used when the block runs stand-alone)."""
        lin = self.emb_layers[1] if which == "t" else self.emb_z_layers[1]
        out = P.new((B, 2 * self.out_channels), torch.float32, "emb_out")
        P.linear(emb, lin.weight, lin.bias, out, B=B, Cin=self.emb_channels, Cout=2 * self.out_channels, a_silu=True)
        return out, 0, 2 * self.out_channels

    # ---- stand-alone forward (NCHW in / NCHW out like the reference) ---------------------------------
    def _forward(self, x, emb, emb_z=None):
        self._check_no_grad(x, emb, emb_z)
        B, C, H, W = x.shape
        key = ("res", B, C, H, W, self.training)

        def build(P: Plan):
            xin = P.new((B, H, W, C), torch.float32, "x_in")
            xin.keep = True
            e = P.new((B, self.emb_channels), torch.float32, "emb_in")
            e.keep = True
            ez = None
            if self.has_z:
                ez = P.new((B, self.emb_channels), torch.float32, "embz_in")
                ez.keep = True
            # touch inputs so they are allocated before the first op
            y = self.emit(P, Src(xin, C, B, H, W), self.emit_emb(P, e, B, "t"),
                          self.emit_emb(P, ez, B, "z") if self.has_z else None)
            y.b1.keep = True
            return xin, e, ez, y

        plan, (xin, e, ez, y) = self._get_plan(key, build)
        xin.tensor.copy_(x.permute(0, 2, 3, 1))
        e.tensor.copy_(emb)
        if self.has_z:
            ez.tensor.copy_(emb_z)
        plan.run()
        return y.b1.tensor.float().permute(0, 3, 1, 2).contiguous()


class ResBlock(_ResBase, TimestepBlock):
    """model/module.py:205-297."""
    has_z = False

    def forward(self, x, emb):
        return self._forward(x, emb)


class ResBlockShift(_ResBase, TimestepContextBlock):
    """model/module.py:299-384: ResBlock + z-conditioned scale/shift ``(1+zs)*(GN(h)*(1+s)+sh)+zsh``."""
    has_z = True

    def forward(self, x, emb, emb_z):
        return self._forward(x, emb, emb_z)


class QKVAttentionLegacy(nn.Module):
    """Marker for the heads-first channel split (model/module.py:431-457)."""

    def __init__(self, n_heads):
        super().__init__()
        self.n_heads = n_heads


class QKVAttention(nn.Module):
    """Marker for the qkv-first channel split (model/module.py:460-488)."""

    def __init__(self, n_heads):
        super().__init__()
        self.n_heads = n_heads


class AttentionBlock(PlannedModule):
    """model/module.py:387-428: GN -> qkv 1x1 -> softmax(QK^T ch^-1/2) V -> proj 1x1 -> + x."""

    def __init__(self, channels, num_heads=1, num_head_channels=-1, use_new_attention_order=False):
        super().__init__()
        self.channels = channels
        if num_head_channels == -1:
            self.num_heads = num_heads
        else:
            assert channels % num_head_channels == 0, \
                f"q,k,v channels {channels} is not divisible by num_head_channels {num_head_channels}"
            self.num_heads = channels // num_head_channels
        self.norm = normalization(channels)
        self.qkv = conv_nd(1, channels, channels * 3, 1)
        self.attention = QKVAttention(self.num_heads) if use_new_attention_order else QKVAttentionLegacy(self.num_heads)
        self.proj_out = zero_module(conv_nd(1, channels, channels, 1))

    def emit(self, P: Plan, x: Src, tape: Optional[list] = None) -> Src:
        assert x.b2 is None and x.C == self.channels
        B, H, W, C = x.B, x.H, x.W, x.C
        T = H * W
        legacy = isinstance(self.attention, QKVAttentionLegacy)
        ab = P.gn_coef(x.b1, C, None, 0, self.norm.weight, self.norm.bias, B=B, HW=T, stats1=x.s1)
        sums = P.last_sums
        tcq = P.use_tc(C, 3 * C, 1, 1, H, W)
        heads, ch = self.num_heads, C // self.num_heads
        # bf16 training forward (autocast): an eligible block runs the bf16 tensor-core attention below and keeps its bf16 qkv,
        # probabilities and attention output for the tensor-core backward (train.Backward.attention)
        amp = tape is not None and P.train_tc == "bf16" and self.amp_eligible(T, ch)
        xn, _ = P.gn_apply(x.b1, C, None, 0, ab, silu=False, resample=RESAMPLE_NONE, B=B, H=H, W=W,
                           act_dtype=torch.bfloat16 if (tcq or amp) else torch.float32)
        if amp or (tcq and P.can_gemm_tc(T, T, ch) and P.can_gemm_tc(T, ch, T)):
            # ---- tensor-core attention: bf16 qkv -> S = Q K^T (batched wgmma GEMM) -> softmax -> P V ----
            qkv = P.new((B, T, 3 * C), torch.bfloat16, "qkv")
            P.conv(xn, self.qkv.weight, self.qkv.bias, qkv, B=B, H=H, W=W, Cin=C, Cout=3 * C, k=1)
            vT = P.new((B * heads, ch, T), torch.bfloat16, "vT")
            P.call("transpose_v", qkv, vT, B, T, C, heads, int(legacy), _STREAM)
            Pm = P.new((B * heads, T, T), torch.bfloat16, "att_probs")
            # (NHWC-shaped under amp: the backward's weight gradient of proj_out takes it as its bf16 input copy)
            att = P.new((B, H, W, C) if amp else (B, T, C), torch.bfloat16, "att")
            hs_ = 3 * ch if legacy else ch                  # channel stride between heads inside a qkv row
            ko = ch if legacy else C                        # offset of K relative to Q
            alpha = 1.0 / math.sqrt(ch)                     # scale = ch^(-1/4) on both q and k (module.py:449-453)
            fuse_sm = T in (64, 128, 256)
            S = None if fuse_sm else P.new((B * heads, T, T), torch.float32, "att_scores")
            for h in range(heads):
                if fuse_sm:   # a whole score row sits in one accumulator tile: softmax in the GEMM epilogue
                    P.gemm_tc(qkv.at(h * hs_), 3 * C, T * 3 * C, qkv.at(h * hs_ + ko), 3 * C, T * 3 * C,
                              Pm.at(h * T * T), T, heads * T * T, batch=B, M=T, N=T, K=ch, out_dtype=torch.bfloat16,
                              softmax_alpha=alpha)
                else:
                    P.gemm_tc(qkv.at(h * hs_), 3 * C, T * 3 * C, qkv.at(h * hs_ + ko), 3 * C, T * 3 * C,
                              S.at(h * T * T), T, heads * T * T, batch=B, M=T, N=T, K=ch, out_dtype=torch.float32)
            if not fuse_sm:
                P.call("softmax_bf16", S, Pm, ctypes.c_int64(B * heads * T), T, ctypes.c_float(alpha), _STREAM)
            for h in range(heads):
                P.gemm_tc(Pm.at(h * T * T), T, heads * T * T, vT.at(h * ch * T), T, heads * ch * T,
                          att.at(h * ch), C, T * C, batch=B, M=T, N=ch, K=T, out_dtype=torch.bfloat16)
            if amp:
                tape.append(("attn", self, dict(x=x, ab=ab, sums=sums, xn=xn, qkv=qkv, probs=Pm, att=att, legacy=legacy,
                                                tc=True)))
        elif tcq and tape is None and P.can_gemm_x3(T, T, ch) and P.can_gemm_x3(T, ch, T):
            # ---- split-operand tensor-core attention (fp32-grade): fp32 qkv -> [hi|lo|hi] x [hi|hi|lo] operand blocks ->
            # S = Q K^T (fp32) -> fp32 softmax, split -> A = P V (fp32); every product is three bf16 wgmma MMAs ----
            qkv = P.new((B, T, 3 * C), torch.float32, "qkv")
            P.conv(xn, self.qkv.weight, self.qkv.bias, qkv, B=B, H=H, W=W, Cin=C, Cout=3 * C, k=1)
            Z = B * heads
            Q3 = P.new((Z, T, 3 * ch), torch.bfloat16, "q3")
            K3 = P.new((Z, T, 3 * ch), torch.bfloat16, "k3")
            VT3 = P.new((Z, ch, 3 * T), torch.bfloat16, "vT3")
            P.call("qkv_split3", qkv, Q3, K3, VT3, B, T, C, heads, int(legacy), _STREAM)
            S = P.new((Z, T, T), torch.float32, "att_scores")
            P.gemm_tc(Q3, 3 * ch, T * 3 * ch, K3, 3 * ch, T * 3 * ch, S, T, T * T, batch=Z, M=T, N=T, K=3 * ch,
                      out_dtype=torch.float32, flops=2.0 * Z * T * T * ch)
            P3 = P.new((Z, T, 3 * T), torch.bfloat16, "att_probs3")
            P.call("softmax_split3", S, P3, ctypes.c_int64(Z * T), T, ctypes.c_float(1.0 / math.sqrt(ch)), _STREAM)
            att = P.new((B, T, C), torch.float32, "att")
            for h in range(heads):
                P.gemm_tc(P3.at(h * T * 3 * T), 3 * T, heads * T * 3 * T, VT3.at(h * ch * 3 * T), 3 * T, heads * ch * 3 * T,
                          att.at(h * ch), C, T * C, batch=B, M=T, N=ch, K=3 * T, out_dtype=torch.float32,
                          flops=2.0 * B * T * ch * T)
            att, _ = P.gn_apply(att, C, None, 0, None, silu=False, resample=RESAMPLE_NONE, B=B, H=H, W=W,
                                act_dtype=torch.bfloat16)
        else:
            qkv = P.new((B, T, 3 * C), torch.float32, "qkv")
            P.conv(xn, self.qkv.weight, self.qkv.bias, qkv, B=B, H=H, W=W, Cin=C, Cout=3 * C, k=1)
            att = P.new((B, T, C), torch.float32, "att")
            scratch = P.new((B * self.num_heads, T, T), torch.float32, "att_scores")
            P.call("attention_simt", qkv, att, scratch, B, T, C, self.num_heads, int(legacy), _STREAM, flops=4.0 * B * T * T * C)
            if tape is not None:
                tape.append(("attn", self, dict(x=x, ab=ab, sums=sums, xn=xn, qkv=qkv, probs=scratch, att=att, legacy=legacy)))
            tcp = P.use_tc(C, C, 1, 1, H, W)
            if tcp:
                att, _ = P.gn_apply(att, C, None, 0, None, silu=False, resample=RESAMPLE_NONE, B=B, H=H, W=W,
                                    act_dtype=torch.bfloat16)
        out = P.new((B, H, W, C), x.b1.dtype if att.dtype == torch.bfloat16 else torch.float32, "attn_out")
        os_ = P.conv(att, self.proj_out.weight, self.proj_out.bias, out, B=B, H=H, W=W, Cin=C, Cout=C, k=1, residual=x.b1,
                     want_stats=True)
        return Src(out, C, B, H, W, s1=os_)

    @staticmethod
    def amp_eligible(T: int, ch: int) -> bool:
        """Does a block with T positions and ch channels per head train on the bf16 tensor-core attention under autocast?
        T % 128 == 0 and T <= 256: a whole score row fits the softmax and softmax-gradient epilogues; ch % 64 == 0: whole k-blocks."""
        return T % 128 == 0 and T <= 256 and ch % 64 == 0

    def forward(self, x):
        self._check_no_grad(x)
        shape = x.shape
        B, C = shape[0], shape[1]
        T = 1
        for s in shape[2:]:
            T *= s
        H, W = (shape[2], shape[3]) if len(shape) == 4 else (1, T)
        key = ("attn", B, C, H, W)

        def build(P: Plan):
            xin = P.new((B, H, W, C), torch.float32, "x_in")
            xin.keep = True
            y = self.emit(P, Src(xin, C, B, H, W))
            y.b1.keep = True
            return xin, y

        plan, (xin, y) = self._get_plan(key, build)
        xin.tensor.copy_(x.reshape(B, C, H, W).permute(0, 2, 3, 1))
        plan.run()
        return y.b1.tensor.float().permute(0, 3, 1, 2).reshape(shape).contiguous()


class TimestepSequential(nn.Sequential, TimestepBlock, TimestepContextBlock):
    """model/module.py:131-140 (dispatch by block type), in plan-emission form."""

    def emit(self, P: Plan, x, emb_of, embz_of=None, tape: Optional[list] = None) -> Src:
        for layer in self:
            if isinstance(layer, ResBlockShift):
                x = layer.emit(P, x, emb_of(layer), embz_of(layer), tape=tape)
            elif isinstance(layer, ResBlock):
                x = layer.emit(P, x, emb_of(layer), tape=tape)
            elif isinstance(layer, AttentionBlock):
                x = layer.emit(P, x, tape=tape)
            else:
                raise TypeError(f"unexpected layer {type(layer).__name__} in TimestepSequential")
        return x
