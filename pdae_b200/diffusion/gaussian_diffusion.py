"""GaussianDiffusion with the reference's public surface (diffusion/gaussian_diffusion.py:11-443):
schedules, q_sample, DDPM ancestral steps, losses, DDIM wrappers, latent / manipulation glue.

Schedule algebra runs in fp64 numpy on the host and is stored as fp32 device tables exactly like the
reference (:31-70).  Per-step arithmetic goes through the fused native kernels (pdae_q_sample,
pdae_noise_p_sample, pdae_ddim_step); respaced DDIM objects are cached per style instead of being rebuilt
(with a device->host copy) on every call (:187,192,276,283).
"""
from __future__ import annotations

import math
from functools import partial
from typing import Dict, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from .. import _native
from .ddim import DDIM, _DDPMRunner, _GapRunner, _f32, _ptr, _stream, _t64, graphable


def _beta_schedule(kind: str, T: int) -> np.ndarray:
    if kind == "linear":
        return np.linspace(0.0001, 0.02, T)
    if kind == "cosine":
        f = lambda s: math.cos((s + 0.008) / 1.008 * math.pi / 2) ** 2
        return np.array([min(1 - f((i + 1) / T) / f(i / T), 0.999) for i in range(T)])
    raise NotImplementedError(kind)


class GaussianDiffusion:
    def __init__(self, config, device):
        self.device = device
        self.timesteps = T = config["timesteps"]
        betas = _beta_schedule(config["betas_type"], T)
        alphas = 1.0 - betas
        ac = np.cumprod(alphas, axis=0)
        ac_prev = np.append(1.0, ac[:-1])
        ac_next = np.append(ac[1:], 0.0)
        post_var = betas * (1.0 - ac_prev) / (1.0 - ac)
        snr = ac / (1.0 - ac)
        self.to_torch = to_torch = partial(torch.tensor, dtype=torch.float32, device=device)
        tables = {
            "alphas": alphas, "betas": betas, "alphas_cumprod": ac, "alphas_cumprod_prev": ac_prev,
            "alphas_cumprod_next": ac_next,
            "sqrt_alphas_cumprod": np.sqrt(ac), "sqrt_one_minus_alphas_cumprod": np.sqrt(1.0 - ac),
            "log_one_minus_alphas_cumprod": np.log(1.0 - ac),
            "sqrt_recip_alphas_cumprod": np.sqrt(1.0 / ac), "sqrt_recip_alphas_cumprod_m1": np.sqrt(1.0 / ac - 1.0),
            "posterior_variance": post_var,
            # clipped: the posterior variance is 0 at t=0
            "posterior_log_variance_clipped": np.log(np.append(post_var[1], post_var[1:])),
            "x_0_posterior_mean_x_0_coef": betas * np.sqrt(ac_prev) / (1.0 - ac),
            "x_0_posterior_mean_x_t_coef": (1.0 - ac_prev) * np.sqrt(alphas) / (1.0 - ac),
            "noise_posterior_mean_x_t_coef": np.sqrt(1.0 / alphas),
            "noise_posterior_mean_noise_coef": betas / (np.sqrt(alphas) * np.sqrt(1.0 - ac)),
            "shift_coef": -np.sqrt(alphas) * (1.0 - ac_prev) / np.sqrt(1.0 - ac),
            "weight": snr ** 0.1 / (1.0 + snr),
        }
        for k, v in tables.items():
            setattr(self, k, to_torch(v))
        self._log_betas = None
        self._ddim_cache: Dict[Tuple[str, int], DDIM] = {}

    # ---- helpers ------------------------------------------------------------------------------------
    # Random draws of the sampling / training glue go through these three methods (same distributions and call order as
    # the reference's torch.randn / randn_like / rand_like calls), so a parity test can substitute a seeded CPU stream.
    def _randn(self, shape):
        return torch.randn(tuple(shape), device=self.device)

    def _randn_like(self, x):
        return torch.randn_like(x)

    def _rand_like(self, x):
        return torch.rand_like(x)

    @staticmethod
    def extract_coef_at_t(schedule, t, x_shape):
        return torch.gather(schedule, -1, t).reshape([x_shape[0]] + [1] * (len(x_shape) - 1))

    @staticmethod
    def get_ddim_betas_and_timestep_map(ddim_style, original_alphas_cumprod):
        """Respacing (:76-94): keep the timesteps int(linspace(0, T-1, S+1)); beta'_k = 1 - abar_k / abar_{k-1}."""
        T = original_alphas_cumprod.shape[0]
        S = int(ddim_style[len("ddim"):])
        keep = sorted(set(int(s) for s in np.linspace(0, T - 1, S + 1)))
        kept = np.asarray(original_alphas_cumprod)[keep]
        # scalar arithmetic of the reference loop: 1 - a / last, `last` starting as the python float 1.0 and
        # then being the previous kept value (so the dtype follows the caller's array: fp32 from `.cpu().numpy()`)
        new_betas = np.array([1 - a / l for a, l in zip(kept, [1.0] + list(kept[:-1]))])
        return new_betas, torch.tensor(keep, dtype=torch.long)

    def _ddim(self, ddim_style, alphas_cumprod=None) -> DDIM:
        src = self.alphas_cumprod if alphas_cumprod is None else alphas_cumprod
        key = (ddim_style, src.data_ptr())
        d = self._ddim_cache.get(key)
        if d is None:
            nb, tmap = self.get_ddim_betas_and_timestep_map(ddim_style, src.cpu().numpy())
            d = DDIM(nb, tmap, self.device)
            self._ddim_cache[key] = d
        return d

    def _ew(self, fn, *args):
        _native.check(fn(*args), fn.__name__ if hasattr(fn, "__name__") else "native elementwise")

    # ---- forward process / posteriors ------------------------------------------------------------------
    def q_sample(self, x_0, t, noise):
        """sqrt(abar_t) x_0 + sqrt(1 - abar_t) noise (:98-103)."""
        if not x_0.is_cuda:
            raise _native.NativeError("q_sample: CUDA tensors required (no CPU fallback)")
        x_0, noise = _f32(x_0), _f32(noise)
        B = x_0.shape[0]
        t = _t64(t, B, "q_sample")
        if noise.shape != x_0.shape:
            raise ValueError(f"q_sample: x_0 {tuple(x_0.shape)} and noise {tuple(noise.shape)} must have one shape")
        out = torch.empty_like(x_0)
        rc = _native.lib().pdae_q_sample(_ptr(x_0), _ptr(noise), _ptr(t), _ptr(self.sqrt_alphas_cumprod),
                                         _ptr(self.sqrt_one_minus_alphas_cumprod), _ptr(out), B, x_0.numel() // B,
                                         _stream(x_0.device))
        _native.check(rc, "pdae_q_sample")
        return out

    def q_posterior_mean(self, x_0, x_t, t):
        s = x_t.shape
        return self.extract_coef_at_t(self.x_0_posterior_mean_x_0_coef, t, s) * x_0 + \
            self.extract_coef_at_t(self.x_0_posterior_mean_x_t_coef, t, s) * x_t

    def noise_p_sample(self, x_t, t, predicted_noise, learned_range=None, noise=None):
        """DDPM ancestral step (:112-126).  ``noise`` defaults to torch.randn(shape) like the reference."""
        if noise is None:
            noise = self._randn(x_t.shape)
        x_t, eps, noise = _f32(x_t), _f32(predicted_noise), _f32(noise)
        lr = _f32(learned_range)
        if lr is not None and self._log_betas is None:
            self._log_betas = torch.log(self.betas)
        B = x_t.shape[0]
        t = _t64(t, B, "noise_p_sample")
        out = torch.empty_like(x_t)
        rc = _native.lib().pdae_noise_p_sample(_ptr(x_t), _ptr(eps), _ptr(noise), _ptr(lr), _ptr(t),
                                               _ptr(self.noise_posterior_mean_x_t_coef),
                                               _ptr(self.noise_posterior_mean_noise_coef),
                                               _ptr(self.posterior_log_variance_clipped), _ptr(self._log_betas), _ptr(out),
                                               B, x_t.numel() // B, _stream(x_t.device))
        _native.check(rc, "pdae_noise_p_sample")
        return out

    def learned_range_to_log_variance(self, learned_range, t):
        s = learned_range.shape
        lo = self.extract_coef_at_t(self.posterior_log_variance_clipped, t, s)
        hi = self.extract_coef_at_t(torch.log(self.betas), t, s)
        return lo + (learned_range + 1) / 2 * (hi - lo)

    def x_0_clip_p_sample(self, x_t, t, predicted_noise, learned_range=None, clip_x_0=True):
        """(:130-146) -- unused by every reference caller; kept for surface completeness (torch elementwise)."""
        s = x_t.shape
        x0 = self.predicted_noise_to_predicted_x_0(x_t, t, predicted_noise)
        if clip_x_0:
            x0 = x0.clamp(-1, 1)
        mean = self.q_posterior_mean(x0, x_t, t)
        logvar = self.learned_range_to_log_variance(learned_range, t) if learned_range is not None else \
            self.extract_coef_at_t(self.posterior_log_variance_clipped, t, s)
        mask = (1 - (t == 0).float()).reshape([s[0]] + [1] * (len(s) - 1))
        return mean + mask * (0.5 * logvar).exp() * self._randn(s)

    def predicted_noise_to_predicted_x_0(self, x_t, t, predicted_noise):
        s = x_t.shape
        return self.extract_coef_at_t(self.sqrt_recip_alphas_cumprod, t, s) * x_t - \
            self.extract_coef_at_t(self.sqrt_recip_alphas_cumprod_m1, t, s) * predicted_noise

    def predicted_noise_to_predicted_mean(self, x_t, t, predicted_noise):
        s = x_t.shape
        return self.extract_coef_at_t(self.noise_posterior_mean_x_t_coef, t, s) * x_t - \
            self.extract_coef_at_t(self.noise_posterior_mean_noise_coef, t, s) * predicted_noise

    def p_loss(self, noise, predicted_noise, weight=None, loss_type="l2"):
        d = noise - predicted_noise
        if loss_type == "l1":
            return d.abs().mean()
        if loss_type == "l2":
            return torch.mean(d ** 2 if weight is None else weight * d ** 2)
        raise NotImplementedError(loss_type)

    # ---- pre-trained DPM / regular DPM ---------------------------------------------------------------
    def test_pretrained_dpms(self, ddim_style, denoise_fn, x_T, condition=None):
        return self.ddim_sample(ddim_style, denoise_fn, x_T, condition)

    def ddim_sample(self, ddim_style, denoise_fn, x_T, condition=None):
        return self._ddim(ddim_style).ddim_sample_loop(denoise_fn, x_T, condition)

    def ddim_encode(self, ddim_style, denoise_fn, x_0, condition=None):
        return self._ddim(ddim_style).ddim_encode_loop(denoise_fn, x_0, condition)

    def regular_train_one_batch(self, denoise_fn, x_0, condition=None):
        B = x_0.shape[0]
        t = torch.randint(0, self.timesteps, (B,), device=self.device, dtype=torch.long)
        noise = self._randn_like(x_0)
        pred = denoise_fn(self.q_sample(x_0=x_0, t=t, noise=noise), t, condition)
        return {"prediction_loss": self.p_loss(noise, pred)}

    def regular_ddim_sample(self, ddim_style, denoise_fn, x_T, condition=None):
        return self.ddim_sample(ddim_style, denoise_fn, x_T, condition)

    def _split_sigma(self, output, C):
        if output.shape[1] == 2 * C:
            return torch.split(output, C, dim=1)
        return output, None

    def identity_map(self):
        """arange(T) on the device: the timestep map of the DDPM loops' device-side step counter (t_loc = t_net = i)."""
        m = self.__dict__.get("_identity_map")
        if m is None:
            with torch.inference_mode(False):
                m = torch.arange(self.timesteps, dtype=torch.int64, device=self.device)
            self.__dict__["_identity_map"] = m
        return m

    def _ddpm_graphed(self, net, x_T, cond, shift):
        """A DDPM loop on the one-graph-per-step path (ddim._DDPMRunner): the network's static plan buffers are driven in
        place; per step the host draws the noise exactly as the generic loop does (self._randn, once per step, same order),
        copies it into the step's static noise buffer and replays the graph."""
        B, C, H, W = x_T.shape
        if shift:
            plan, (x_in, t_in, z_in, eps, grad) = net.plan_for(B, H, W)
            z_in.tensor.copy_(cond)
        else:
            plan, (x_in, t_in, c_in, eps) = net.plan_for(B, H, W)
            grad = None
            if c_in is not None:
                c_in.tensor.copy_(cond)
        run = _DDPMRunner(self, plan, x_in, t_in, eps, grad, C)
        run.begin()
        try:
            x_in.tensor.copy_(x_T)
            run.seek(self.timesteps - 1)
            for _ in range(self.timesteps):
                run.noise.copy_(self._randn(x_T.shape))
                run.step()
            return x_in.tensor.clone()
        finally:
            run.end()

    def regular_ddpm_sample(self, denoise_fn, x_T, condition=None):
        from ..model.unet import UNet
        if isinstance(denoise_fn, UNet) and graphable(denoise_fn, x_T):
            return self._ddpm_graphed(denoise_fn, x_T, condition, shift=False)
        B, C = x_T.shape[0], x_T.shape[1]
        img = x_T
        for i in reversed(range(self.timesteps)):
            t = torch.full((B,), i, device=self.device, dtype=torch.long)
            eps, lr = self._split_sigma(denoise_fn(img, t, condition), C)
            img = self.noise_p_sample(img, t, eps, lr)
        return img

    # ---- representation learning (PDAE) ----------------------------------------------------------------
    def representation_learning_train_one_batch(self, encoder, decoder, x_0):
        s = x_0.shape
        z = encoder(x_0)
        t = torch.randint(0, self.timesteps, (s[0],), device=self.device, dtype=torch.long)
        noise = self._randn_like(x_0)
        eps, grad = decoder(self.q_sample(x_0=x_0, t=t, noise=noise), t, z)
        target = eps + self.extract_coef_at_t(self.shift_coef, t, s) * grad
        return {"prediction_loss": self.p_loss(noise, target, weight=self.extract_coef_at_t(self.weight, t, s))}

    def representation_learning_ddpm_sample(self, encoder, decoder, x_0, x_T, z=None):
        s = x_0.shape
        if z is None:
            z = encoder(x_0)
        from ..model.shift_unet import ShiftUNet
        if (isinstance(decoder, ShiftUNet) and graphable(decoder, x_T) and s[0] == x_T.shape[0]
                and decoder.output_channel == x_T.shape[1]):   # (learned sigma: eps + coef * grad does not broadcast)
            return self._ddpm_graphed(decoder, x_T, z, shift=True)
        img = x_T
        for i in reversed(range(self.timesteps)):
            t = torch.full((s[0],), i, device=self.device, dtype=torch.long)
            eps, grad = decoder(img, t, z)
            img = self.noise_p_sample(img, t, eps + self.extract_coef_at_t(self.shift_coef, t, s) * grad)
        return img

    def representation_learning_ddim_sample(self, ddim_style, encoder, decoder, x_0, x_T, z=None, stop_percent=0.0):
        if z is None:
            z = encoder(x_0)
        return self._ddim(ddim_style).shift_ddim_sample_loop(decoder, z, x_T, stop_percent=stop_percent)

    def representation_learning_ddim_encode(self, ddim_style, encoder, decoder, x_0, z=None):
        if z is None:
            z = encoder(x_0)
        return self._ddim(ddim_style).shift_ddim_encode_loop(decoder, z, x_0)

    def representation_learning_autoencoding(self, encoder_ddim_style, decoder_ddim_style, encoder, decoder, x_0):
        z = encoder(x_0)
        x_T = self.representation_learning_ddim_encode(encoder_ddim_style, encoder, decoder, x_0, z)
        return self.representation_learning_ddim_sample(decoder_ddim_style, None, decoder, None, x_T, z)

    def _gap_graphed(self, decoder, x_0, z):
        """The gap measure on the one-graph-per-step path (ddim._GapRunner): x_0 and z are written once into static buffers;
        per step the host draws the uniform noise exactly as the generic loop does (self._rand_like, once per step, same
        order), copies it into the step's static noise buffer and replays the graph.  The [T][2] results reach the host once."""
        B, C, H, W = x_0.shape
        plan, (x_in, t_in, z_in, eps, grad) = decoder.plan_for(B, H, W)
        z_in.tensor.copy_(z)
        run = _GapRunner(self, plan, x_in, t_in, eps, grad, C)
        run.x0.copy_(_f32(x_0))
        run.begin()
        try:
            run.seek(self.timesteps - 1)
            for _ in range(self.timesteps):
                run.noise.copy_(self._rand_like(x_0))
                run.step()
            gaps = run.gaps.cpu().flip(0)          # row t -> the reference's order t = T-1 .. 0
        finally:
            run.end()
        return gaps[:, 0].tolist(), gaps[:, 1].tolist()

    def representation_learning_gap_measure(self, encoder, decoder, x_0):
        """(:292-318) -- NB the reference draws its 'noise' with torch.rand_like (uniform); kept.
        On a pdae_b200 ShiftUNet (grad off, epsilon-only output) a step is one CUDA graph and the gaps are reduced on the
        device (_gap_graphed); any other decoder takes the generic loop below."""
        s = x_0.shape
        z = encoder(x_0)
        from ..model.shift_unet import ShiftUNet
        if isinstance(decoder, ShiftUNet) and graphable(decoder, x_0) and decoder.output_channel == s[1]:
            return self._gap_graphed(decoder, x_0, z)
        gap_pred, gap_ae = [], []
        for i in reversed(range(self.timesteps)):
            t = torch.full((s[0],), i, device=self.device, dtype=torch.long)
            x_t = self.q_sample(x_0, t, self._rand_like(x_0))
            eps, grad = decoder(x_t, t, z)
            true_mean = self.q_posterior_mean(x_0, x_t, t)
            m1 = self.q_posterior_mean(self.predicted_noise_to_predicted_x_0(x_t, t, eps), x_t, t)
            eps_ae = eps + self.extract_coef_at_t(self.shift_coef, t, s) * grad
            m2 = self.q_posterior_mean(self.predicted_noise_to_predicted_x_0(x_t, t, eps_ae), x_t, t)
            gap_pred.append(torch.mean((true_mean - m1) ** 2).cpu().item())
            gap_ae.append(torch.mean((true_mean - m2) ** 2).cpu().item())
        return gap_pred, gap_ae

    def representation_learning_denoise_one_step(self, encoder, decoder, x_0, timestep_list):
        s = x_0.shape
        t = torch.tensor(timestep_list, device=self.device, dtype=torch.long)
        x_t = self.q_sample(x_0, t, noise=self._randn_like(x_0))
        eps, grad = decoder(x_t, t, encoder(x_0))
        eps_ae = eps + self.extract_coef_at_t(self.shift_coef, t, s) * grad
        return self.predicted_noise_to_predicted_x_0(x_t, t, eps), self.predicted_noise_to_predicted_x_0(x_t, t, eps_ae)

    def representation_learning_ddim_trajectory_interpolation(self, ddim_style, decoder, z_1, z_2, x_T, alpha):
        return self._ddim(ddim_style).shift_ddim_trajectory_interpolation(decoder, z_1, z_2, x_T, alpha)

    # ---- latent DPM ----------------------------------------------------------------------------------
    @property
    def latent_diffusion_config(self):
        """Constant beta = 0.008, T = 1000, L1 loss (:344-363); tables cached."""
        cfg = self.__dict__.get("_latent_cfg")
        if cfg is None:
            T = 1000
            betas = np.array([0.008] * T)
            ac = np.cumprod(1.0 - betas, axis=0)
            cfg = {"timesteps": T, "betas": betas, "alphas_cumprod": self.to_torch(ac),
                   "sqrt_alphas_cumprod": self.to_torch(np.sqrt(ac)),
                   "sqrt_one_minus_alphas_cumprod": self.to_torch(np.sqrt(1.0 - ac)), "loss_type": "l1"}
            self.__dict__["_latent_cfg"] = cfg
        return cfg

    def normalize(self, z, mean, std):
        return (z - mean) / std

    def denormalize(self, z, mean, std):
        return z * std + mean

    def latent_diffusion_train_one_batch(self, latent_denoise_fn, encoder, x_0, latents_mean, latents_std):
        cfg = self.latent_diffusion_config
        z_0 = self.normalize(encoder(x_0).detach(), latents_mean, latents_std)
        s = z_0.shape
        t = torch.randint(0, cfg["timesteps"], (s[0],), device=self.device, dtype=torch.long)
        noise = self._randn_like(z_0)
        z_t = self.extract_coef_at_t(cfg["sqrt_alphas_cumprod"], t, s) * z_0 + \
            self.extract_coef_at_t(cfg["sqrt_one_minus_alphas_cumprod"], t, s) * noise
        return {"prediction_loss": self.p_loss(noise, latent_denoise_fn(z_t, t), loss_type=cfg["loss_type"])}

    def latent_diffusion_sample(self, latent_ddim_style, decoder_ddim_style, latent_denoise_fn, decoder, x_T, latents_mean,
                                latents_std):
        z_T = self._randn((x_T.shape[0], latent_denoise_fn.input_channel))
        z_T.clamp_(-1.0, 1.0)  # as in the reference: "may slightly improve sample quality"
        z = self._ddim(latent_ddim_style, self.latent_diffusion_config["alphas_cumprod"]).latent_ddim_sample_loop(
            latent_denoise_fn, z_T)
        z = self.denormalize(z, latents_mean, latents_std)
        return self.representation_learning_ddim_sample(decoder_ddim_style, None, decoder, None, x_T, z, stop_percent=0.3)

    # ---- manipulation -----------------------------------------------------------------------------------
    def manipulation_train_one_batch(self, classifier, encoder, x_0, label, latents_mean, latents_std):
        z_norm = self.normalize(encoder(x_0).detach(), latents_mean, latents_std)
        gt = (label > 0).float()
        return {"bce_loss": F.binary_cross_entropy_with_logits(classifier(z_norm), gt)}

    def manipulation_sample(self, ddim_style, classifier_weight, encoder, decoder, x_0, inferred_x_T, latents_mean,
                            latents_std, class_id, scale):
        z_norm = self.normalize(encoder(x_0), latents_mean, latents_std)
        direction = F.normalize(classifier_weight[class_id][None, :], dim=1)
        z = self.denormalize(z_norm + scale * math.sqrt(512) * direction, latents_mean, latents_std)
        return self.representation_learning_ddim_sample(ddim_style, None, decoder, None, inferred_x_T, z, stop_percent=0.0)
