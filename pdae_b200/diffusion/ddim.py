"""Respaced deterministic DDIM (reference surface: diffusion/ddim.py:7-207) on native kernels.

Same constructor (``DDIM(betas, timestep_map, device)``) and method names.  The per-step arithmetic
(23 ATen launches in the reference) is ONE fused kernel, ``pdae_ddim_step``; when the network is a
pdae_b200 ShiftUNet/UNet the loop drives the network's static plan buffers directly (no per-step
allocation, no host sync, no tqdm).
"""
from __future__ import annotations

import ctypes
from functools import partial

import numpy as np
import torch

from .. import _native
from ..engine import FUSE_DESC_LEN


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _f32(t):
    """The elementwise kernels read raw fp32 pointers: promote anything else (half tensors under AMP, double images from a
    dataset) the way the reference's type-promoting torch arithmetic would, instead of reinterpreting the bytes."""
    return None if t is None else t.to(torch.float32).contiguous()


def _t64(t, B, what):
    t = t.to(torch.int64).contiguous()
    if t.numel() != B:
        raise ValueError(f"{what}: t must hold one timestep per sample ({B}), got {tuple(t.shape)}")
    return t


def graphable(net, x) -> bool:
    """Does a sampling loop over `net` run on the one-graph-per-step path (a pdae_b200 UNet / ShiftUNet on a 4-D CUDA input,
    or a pdae_b200 MLPSkipNet on a 2-D one, with autograd off)?  Any other callable takes the generic per-step loop."""
    from ..model.mlp_skip_net import MLPSkipNet
    from ..model.shift_unet import ShiftUNet
    from ..model.unet import UNet
    if not x.is_cuda or torch.is_grad_enabled():
        return False
    return (isinstance(net, (ShiftUNet, UNet)) and x.dim() == 4) or (isinstance(net, MLPSkipNet) and x.dim() == 2)


class _StepRunner:
    """One network plan + the loop bookkeeping + the fused update of a DDIM loop direction, replayed as ONE CUDA graph per
    step.  The graph is cached on the plan, keyed by (owner, kind, shift) -- those fix the table pointers the update
    reads; the cache entry keeps the owner (DDIM / GaussianDiffusion object) alive so its id is not reused.  `seek(i)` sets
    the device-side step counter; `step()` is a single graph launch.  _DDPMRunner and _InterpRunner change the update."""

    def __init__(self, ddim, plan, x_in, t_in, eps, grad, direction: str, C: int, tmap=None, key=None):
        self.d, self.plan, self.x_in, self.t_in, self.eps, self.grad, self.direction = ddim, plan, x_in, t_in, eps, grad, direction
        self.tmap = ddim.timestep_map if tmap is None else tmap
        dev = ddim.device
        B = x_in.tensor.shape[0]
        self.B = B
        self.delta = 1 if direction == "encode" else -1
        # the update runs inside the step graph (separate kernel, or fused into the last head conv's epilogue); only a learn_sigma
        # head on the CUDA-core path (2C output channels, no fusable epilogue) needs it after the replay
        self.in_graph_update = eps.tensor.shape[1] == C or bool(getattr(plan, "head_fuse", None))
        self.fused = False
        self.C = C
        cache = plan.__dict__.setdefault("_step_cache", {})
        key = (id(ddim),) + (key or (direction, grad is not None))
        ent = cache.get(key)
        if ent is None:
            with torch.inference_mode(False):   # never inference tensors: the cache outlives the caller's autograd mode
                ent = {"counter": torch.zeros(1, dtype=torch.int64, device=dev),
                       "t_loc": torch.zeros(B, dtype=torch.int64, device=dev), "graph": None, "ddim": ddim}
            cache[key] = ent
        self.ent = ent

    def _fuse_target(self):
        """The image head that ends the step plan and can run the update in its epilogue (tensor-core heads only)."""
        hf = getattr(self.plan, "head_fuse", None) or {}
        if "grad" in hf:
            return hf["grad"], True
        if "eps" in hf:
            return hf["eps"], False
        return None, False

    def _fuse_desc(self, is_grad_head: bool):
        """Descriptor of the update fused into the head's epilogue (include/pdae_b200.h: pdae_conv_tc2_set_head_fuse), or None
        to run the standalone update instead."""
        d = self.d
        tab = d.alphas_cumprod_prev if self.direction == "sample" else d.alphas_cumprod_next
        Ce = int(self.eps.tensor.shape[1])
        flags = 1 | (self.C << 8) | (Ce << 16)
        if is_grad_head:
            flags |= 2 if self.grad is not None else 4
        return [flags, self.eps.tensor.data_ptr(), self.x_in.tensor.data_ptr(), self.ent["t_loc"].data_ptr(),
                d.sqrt_recip_alphas_cumprod.data_ptr(), d.sqrt_recip_alphas_cumprod_m1.data_ptr(),
                d.sqrt_one_minus_alphas_cumprod.data_ptr(), tab.data_ptr()]

    def _update(self):
        """The standalone update, inside the step graph."""
        x = self.x_in.tensor
        self.d._update(x, self.ent["t_loc"], self.eps.tensor, self.grad.tensor if self.grad is not None else None,
                       self.direction, out=x)

    def _select_t(self):
        rc = _native.lib().pdae_ddim_select_t(_ptr(self.ent["counter"]), self.delta, _ptr(self.tmap), int(self.tmap.shape[0]),
                                              _ptr(self.ent["t_loc"]), _ptr(self.t_in.tensor), self.B, _stream(self.d.device))
        _native.check(rc, "pdae_ddim_select_t")

    def _launch_step(self):
        self._select_t()
        self.plan._launch_all()
        if self.in_graph_update and not self.fused:
            self._update()

    def begin(self):
        self.plan.run_prologue()          # forced weight re-pack + step-invariant ops (label_emb(z), emb_z_layers)
        # update fused into the last head conv's epilogue: point its device-side descriptor at this loop's tables
        fuse, is_grad_head = self._fuse_target()
        desc = self._fuse_desc(is_grad_head) if fuse is not None and self.in_graph_update else None
        self.fused = desc is not None
        self.fuse_buf = fuse if self.fused else None
        if self.fused:
            fuse.tensor.copy_(torch.tensor(desc + [0] * (FUSE_DESC_LEN - len(desc)), dtype=torch.int64))
        gkey = "graph_fused" if self.fused else "graph"
        if self.ent.get(gkey) is None:
            self.seek(1 if self.direction == "sample" else 0)
            self._launch_step()           # warm-up outside capture (lazy module loading, cudaFuncSetAttribute, ...)
            torch.cuda.synchronize(self.d.device)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._launch_step()
            self.ent[gkey] = g
        self.graph = self.ent[gkey]

    def end(self):
        """Switch the fused update off again: the plan is shared with plain forward calls."""
        if getattr(self, "fuse_buf", None) is not None:
            self.fuse_buf.tensor.zero_()

    def seek(self, i: int):
        self.ent["counter"].fill_(int(i))

    def step(self):
        self.graph.replay()
        if not self.in_graph_update:
            x = self.x_in.tensor
            e = self.eps.tensor[:, :self.C].contiguous()
            self.d._update(x, self.ent["t_loc"], e, self.grad.tensor if self.grad is not None else None, self.direction, out=x)


class _DDPMRunner(_StepRunner):
    """A DDPM ancestral loop (gaussian_diffusion.py:216-229 regular, :257-270 representation learning) on the step graph:
    the counter runs T-1 .. 0 over the identity map (t_loc = t_net = i); the caller writes each step's N(0, 1) draw into
    `noise` before `step()`.  The update is fused into the last tensor-core head (UNet epsilon head; ShiftUNet shift head,
    eps + shift_coef[t] * grad) or runs as pdae_noise_p_sample_shift inside the graph (fp32 / CUDA-core heads, learned
    sigma: epsilon and log-variance range are the two halves of the 2C output)."""

    def __init__(self, gd, plan, x_in, t_in, eps, grad, C: int):
        super().__init__(gd, plan, x_in, t_in, eps, grad, "ddpm", C, tmap=gd.identity_map(), key=("ddpm", grad is not None))
        self.in_graph_update = True
        if "noise" not in self.ent:
            with torch.inference_mode(False):
                self.ent["noise"] = torch.zeros_like(x_in.tensor)
        self.noise = self.ent["noise"]
        if eps.tensor.shape[1] != C and gd._log_betas is None:
            gd._log_betas = torch.log(gd.betas)

    def _fuse_desc(self, is_grad_head: bool):
        gd, C = self.d, self.C
        if self.eps.tensor.shape[1] != C:       # learned sigma: epsilon and range sit in different lanes of the head
            return None
        flags = 1 | 8 | (2 if self.grad is not None else 0) | (C << 8) | (C << 16)
        return [flags, self.eps.tensor.data_ptr(), self.x_in.tensor.data_ptr(), self.ent["t_loc"].data_ptr(),
                gd.noise_posterior_mean_x_t_coef.data_ptr(), gd.noise_posterior_mean_noise_coef.data_ptr(),
                gd.shift_coef.data_ptr(), gd.posterior_log_variance_clipped.data_ptr(), self.noise.data_ptr()]

    def _update(self):
        gd, x, e = self.d, self.x_in.tensor, self.eps.tensor
        per = x.numel() // self.B
        lr = ctypes.c_void_p(e.data_ptr() + per * e.element_size()) if e.shape[1] != self.C else None
        rc = _native.lib().pdae_noise_p_sample_shift(
            _ptr(x), _ptr(e), _ptr(self.grad.tensor if self.grad is not None else None), _ptr(gd.shift_coef), _ptr(self.noise),
            lr, e.numel() // self.B, _ptr(self.ent["t_loc"]), _ptr(gd.noise_posterior_mean_x_t_coef),
            _ptr(gd.noise_posterior_mean_noise_coef), _ptr(gd.posterior_log_variance_clipped), _ptr(gd._log_betas), _ptr(x),
            self.B, per, _stream(x.device))
        _native.check(rc, "pdae_noise_p_sample_shift")


class _GapRunner(_StepRunner):
    """The gap measure (gaussian_diffusion.py:292-318) on the step graph of a ShiftUNet plan: the counter runs T-1 .. 0 over
    the identity map; a step is pdae_q_sample of the static x_0 and noise buffers into the plan's input, the network, and
    pdae_gap_terms writing both mean squared gaps into row t of the static [T][2] buffer `gaps`.  The caller writes x_0 once
    and each step's uniform draw into `noise` before `step()`.  Nothing is fused into the heads: a plain forward afterwards
    sees the plan unchanged."""

    def __init__(self, gd, plan, x_in, t_in, eps, grad, C: int):
        super().__init__(gd, plan, x_in, t_in, eps, grad, "gap", C, tmap=gd.identity_map(), key=("gap",))
        self.in_graph_update = True
        if "gaps" not in self.ent:
            ws = _native.lib().pdae_gap_terms_workspace_bytes(x_in.tensor.numel())
            if ws < 0:
                _native.check(ws, "pdae_gap_terms_workspace_bytes")
            with torch.inference_mode(False):
                self.ent["x0"] = torch.zeros_like(x_in.tensor)
                self.ent["noise"] = torch.zeros_like(x_in.tensor)
                self.ent["gaps"] = torch.zeros(gd.timesteps, 2, dtype=torch.float32, device=gd.device)
                self.ent["ws"] = torch.empty(ws // 8, dtype=torch.float64, device=gd.device)
        self.x0, self.noise, self.gaps, self.ws = self.ent["x0"], self.ent["noise"], self.ent["gaps"], self.ent["ws"]

    def _fuse_desc(self, is_grad_head: bool):
        return None

    def _launch_step(self):
        L, gd = _native.lib(), self.d
        st = _stream(gd.device)
        t = self.ent["t_loc"]
        self._select_t()
        x = self.x_in.tensor
        per = x.numel() // self.B
        rc = L.pdae_q_sample(_ptr(self.x0), _ptr(self.noise), _ptr(t), _ptr(gd.sqrt_alphas_cumprod),
                             _ptr(gd.sqrt_one_minus_alphas_cumprod), _ptr(x), self.B, per, st)
        _native.check(rc, "pdae_q_sample")
        self.plan._launch_all()
        rc = L.pdae_gap_terms(_ptr(self.x0), _ptr(x), _ptr(self.eps.tensor), _ptr(self.grad.tensor), _ptr(t),
                              _ptr(gd.x_0_posterior_mean_x_0_coef), _ptr(gd.x_0_posterior_mean_x_t_coef),
                              _ptr(gd.sqrt_recip_alphas_cumprod), _ptr(gd.sqrt_recip_alphas_cumprod_m1), _ptr(gd.shift_coef),
                              _ptr(self.ws), self.ws.numel() * 8, _ptr(self.gaps), self.B, per, st)
        _native.check(rc, "pdae_gap_terms")


class _InterpRunner(_StepRunner):
    """DDIM trajectory interpolation (ddim.py:149-174) on ShiftUNet.plan_for_interp: epsilon and the frozen half once, the
    shift half for z_1 and z_2; the update (gradient (1 - alpha) g1 + alpha g2, then the DDIM step) is fused into the second
    shift head or runs as pdae_grad_blend + pdae_ddim_step inside the graph.  alpha lives in device memory (the descriptor,
    `ab`), so one captured graph serves every alpha."""

    def __init__(self, ddim, plan, x_in, t_in, eps, g1, g2, C: int, alpha):
        super().__init__(ddim, plan, x_in, t_in, eps, g2, "sample", C, key=("interp",))
        self.g1 = g1
        if "ab" not in self.ent:
            with torch.inference_mode(False):
                self.ent["ab"] = torch.zeros(2, dtype=torch.float32, device=ddim.device)
                self.ent["g"] = torch.zeros_like(g2.tensor)
        self.ab = np.array([1.0 - alpha, alpha], dtype=np.float32)   # torch's fp32 scalars of (1.0 - alpha) * g1 + alpha * g2

    def begin(self):
        self.ent["ab"].copy_(torch.from_numpy(self.ab))
        super().begin()

    def _fuse_desc(self, is_grad_head: bool):
        desc = super()._fuse_desc(is_grad_head)
        desc[0] |= 16
        return desc + [self.g1.tensor.data_ptr(), int(self.ab.view(np.int64)[0])]

    def _update(self):
        x, g = self.x_in.tensor, self.ent["g"]
        rc = _native.lib().pdae_grad_blend(_ptr(self.g1.tensor), _ptr(self.grad.tensor), _ptr(self.ent["ab"]), _ptr(g),
                                           g.numel(), _stream(x.device))
        _native.check(rc, "pdae_grad_blend")
        self.d._update(x, self.ent["t_loc"], self.eps.tensor, g, "sample", out=x)


class DDIM:
    def __init__(self, betas, timestep_map, device):
        self.device = device
        self.timestep_map = timestep_map.to(self.device)
        self.timesteps = betas.shape[0] - 1
        # fp64 schedule algebra on the host, fp32 tables on the device -- exactly ddim.py:15-33
        acp = np.cumprod(1.0 - betas, axis=0)
        f32 = partial(torch.tensor, dtype=torch.float32, device=self.device)
        self.alphas_cumprod_prev = f32(np.append(1.0, acp[:-1]))
        self.alphas_cumprod_next = f32(np.append(acp[1:], 0.0))
        self.sqrt_one_minus_alphas_cumprod = f32(np.sqrt(1.0 - acp))
        self.sqrt_recip_alphas_cumprod = f32(np.sqrt(1.0 / acp))
        self.sqrt_recip_alphas_cumprod_m1 = f32(np.sqrt(1.0 / acp - 1.0))

    @staticmethod
    def extract_coef_at_t(schedule, t, x_shape):
        return torch.gather(schedule, -1, t).reshape([x_shape[0]] + [1] * (len(x_shape) - 1))

    def t_transform(self, t):
        return self.timestep_map[t]

    # ---- the fused update ---------------------------------------------------------------------------
    def _update(self, x_t, t, eps, grad, direction, out=None):
        if not x_t.is_cuda:
            raise _native.NativeError("DDIM: CUDA tensors required (no CPU fallback)")
        x_t, eps, grad = _f32(x_t), _f32(eps), _f32(grad)
        B = x_t.shape[0]
        t = _t64(t, B, "DDIM update")
        if eps.shape != x_t.shape or (grad is not None and grad.shape != x_t.shape):
            raise ValueError(f"DDIM update: x_t {tuple(x_t.shape)}, eps {tuple(eps.shape)} and grad must have one shape")
        out = torch.empty_like(x_t) if out is None else out
        tab = self.alphas_cumprod_prev if direction == "sample" else self.alphas_cumprod_next
        rc = _native.lib().pdae_ddim_step(_ptr(x_t), _ptr(eps), _ptr(grad), _ptr(t), _ptr(self.sqrt_recip_alphas_cumprod),
                                          _ptr(self.sqrt_recip_alphas_cumprod_m1), _ptr(self.sqrt_one_minus_alphas_cumprod),
                                          _ptr(tab), _ptr(out), B, x_t.numel() // B, _stream(x_t.device))
        _native.check(rc, "pdae_ddim_step")
        return out

    # ---- single steps (ddim.py:43-55, 66-79, 91-107, 123-138) -----------------------------------------
    def ddim_sample(self, denoise_fn, x_t, t, condition=None):
        return self._update(x_t, t, denoise_fn(x_t, self.t_transform(t), condition), None, "sample")

    def ddim_encode(self, denoise_fn, x_t, t, condition=None):
        return self._update(x_t, t, denoise_fn(x_t, self.t_transform(t), condition), None, "encode")

    def shift_ddim_sample(self, decoder, z, x_t, t, use_shift=True):
        eps, grad = decoder(x_t, self.t_transform(t), z)
        return self._update(x_t, t, eps, grad if use_shift else None, "sample")

    def shift_ddim_encode(self, decoder, z, x_t, t):
        eps, grad = decoder(x_t, self.t_transform(t), z)
        return self._update(x_t, t, eps, grad, "encode")

    # ---- loops (ddim.py:57-64, 81-88, 110-120, 140-147) -----------------------------------------------
    def _steps(self, direction):
        return reversed(range(1, self.timesteps + 1)) if direction == "sample" else range(0, self.timesteps)

    def _loop(self, net, x, cond, direction, shift, stop_step=0):
        from ..model.shift_unet import ShiftUNet
        B = x.shape[0]
        ts = torch.arange(0, self.timesteps + 1, device=self.device, dtype=torch.int64)
        if not graphable(net, x) or x.dim() != 4:   # (an MLPSkipNet's graphed loop is latent_ddim_sample_loop)
            img = x
            for i in self._steps(direction):
                t = ts[i].expand(B).contiguous()
                if shift:
                    eps, grad = net(img, self.t_transform(t), cond)
                    img = self._update(img, t, eps, grad if (direction == "encode" or (i - 1) >= stop_step) else None,
                                       direction)
                else:
                    img = self._update(img, t, net(img, self.t_transform(t), cond), None, direction)
            return img
        # fast path: drive the network's static plan buffers in place; a WHOLE step -- loop-index broadcast + timestep
        # map lookup, every network launch, the fused DDIM update writing x_t back into the network's input buffer -- is one
        # CUDA graph (device-side step counter), so a step costs one graph launch and no other host work
        H, W = x.shape[2], x.shape[3]
        C = x.shape[1]
        tail = None   # StepRunner of the epsilon-only plan used once the shift is switched off
        if isinstance(net, ShiftUNet):
            plan, (x_in, t_in, z_in, eps, grad) = net.plan_for(B, H, W)
            z_in.tensor.copy_(cond)
            main = _StepRunner(self, plan, x_in, t_in, eps, grad if shift else None, direction, C)
            if shift and direction == "sample" and stop_step > 0:
                # ddim.py:119: steps with (i-1) < stop_step ignore the shift -> replay only the frozen epsilon half there
                p2, (x2, t2, _, eps2, _) = net.plan_for(B, H, W, with_shift=False)
                tail = _StepRunner(self, p2, x2, t2, eps2, None, direction, C)
        else:
            plan, (x_in, t_in, c_in, eps) = net.plan_for(B, H, W)
            if c_in is not None:
                c_in.tensor.copy_(cond)
            main = _StepRunner(self, plan, x_in, t_in, eps, None, direction, C)
        main.begin()   # re-packs weights (forced: `.data` / raw-pointer updates bump no version), prologue
        if tail is not None:
            tail.begin()
        try:
            x_in.tensor.copy_(x)
            cur = main
            steps = list(self._steps(direction))
            cur.seek(steps[0])
            for i in steps:
                use_shift = shift and (direction == "encode" or (i - 1) >= stop_step)
                if tail is not None and not use_shift and cur is not tail:
                    tail.x_in.tensor.copy_(cur.x_in.tensor)
                    cur = tail
                    cur.seek(i)
                cur.step()
            return cur.x_in.tensor.clone()
        finally:
            main.end()
            if tail is not None:
                tail.end()

    def ddim_sample_loop(self, denoise_fn, x_T, condition=None):
        return self._loop(denoise_fn, x_T, condition, "sample", shift=False)

    def ddim_encode_loop(self, denoise_fn, x_0, condition=None):
        return self._loop(denoise_fn, x_0, condition, "encode", shift=False)

    def shift_ddim_sample_loop(self, decoder, z, x_T, stop_percent=0.0):
        return self._loop(decoder, x_T, z, "sample", shift=True, stop_step=int(stop_percent * self.timesteps))

    def shift_ddim_encode_loop(self, decoder, z, x_0):
        return self._loop(decoder, x_0, z, "encode", shift=True)

    def shift_ddim_trajectory_interpolation(self, decoder, z_1, z_2, x_T, alpha):
        """ddim.py:149-174: two decoder calls per step, gradient = (1-alpha) g1 + alpha g2, epsilon from the first.
        On a ShiftUNet a step is one graph of the interpolation plan: the frozen half (and epsilon) is evaluated once, only
        the shift half runs for both z (ShiftUNet.plan_for_interp)."""
        from ..model.shift_unet import ShiftUNet
        B = x_T.shape[0]
        if (isinstance(decoder, ShiftUNet) and graphable(decoder, x_T)
                and decoder.output_channel == x_T.shape[1]):   # (learned sigma: the generic loop raises)
            _, C, H, W = x_T.shape
            plan, (x_in, t_in, z1_in, z2_in, eps, g1, g2) = decoder.plan_for_interp(B, H, W)
            z1_in.tensor.copy_(z_1)
            z2_in.tensor.copy_(z_2)
            run = _InterpRunner(self, plan, x_in, t_in, eps, g1, g2, C, alpha)
            run.begin()
            try:
                x_in.tensor.copy_(x_T)
                run.seek(self.timesteps)
                for _ in range(self.timesteps):
                    run.step()
                return x_in.tensor.clone()
            finally:
                run.end()
        x_t = x_T
        for i in reversed(range(1, self.timesteps + 1)):
            t = torch.full((B,), i, device=self.device, dtype=torch.long)
            eps, g1 = decoder(x_t, self.t_transform(t), z_1)
            _, g2 = decoder(x_t, self.t_transform(t), z_2)
            x_t = self._update(x_t, t, eps, (1.0 - alpha) * g1 + alpha * g2, "sample")
        return x_t

    def latent_ddim_sample(self, latent_denoise_fn, z_t, t):
        """ddim.py:178-198 -- the unclamped single step (no caller in the reference uses it: its loop goes through
        ddim_sample).  z_0 = A_t z_t - B_t eps;  z_prev = sqrt(abar_prev) z_0 + sqrt(1 - abar_prev) eps."""
        s = z_t.shape
        eps = latent_denoise_fn(z_t, self.t_transform(t))
        z0 = self.extract_coef_at_t(self.sqrt_recip_alphas_cumprod, t, s) * z_t - \
            self.extract_coef_at_t(self.sqrt_recip_alphas_cumprod_m1, t, s) * eps
        ap = self.extract_coef_at_t(self.alphas_cumprod_prev, t, s)
        return z0 * torch.sqrt(ap) + torch.sqrt(1.0 - ap) * eps

    def latent_ddim_sample_loop(self, latent_denoise_fn, z_T):
        """ddim.py:200-207 -- NB calls ddim_sample, i.e. WITH the clamp of the predicted z_0.
        On a pdae_b200 MLPSkipNet a step is one graph: the timestep lookup, the network's plan for a batch that shares its
        timestep (MLPSkipNet.plan_for(B, one_t=True)) and the clamped update written back into the plan's z_t input."""
        from ..model.mlp_skip_net import MLPSkipNet
        B = z_T.shape[0]
        if isinstance(latent_denoise_fn, MLPSkipNet) and graphable(latent_denoise_fn, z_T):
            plan, (x_in, t_in, eps) = latent_denoise_fn.plan_for(B, one_t=True)
            run = _StepRunner(self, plan, x_in, t_in, eps, None, "sample", z_T.shape[1], key=("latent",))
            run.begin()
            try:
                x_in.tensor.copy_(z_T)
                run.seek(self.timesteps)
                for _ in range(self.timesteps):
                    run.step()
                return x_in.tensor.clone()
            finally:
                run.end()
        z = z_T
        for i in reversed(range(1, self.timesteps + 1)):
            t = torch.full((B,), i, device=self.device, dtype=torch.long)
            z = self.ddim_sample(latent_denoise_fn, z, t)
        return z
