"""pdae_b200 -- Hopper-native (H100, sm_90a) implementation of the PDAE hot path.

Public surface mirrors the reference repo's modules:
    pdae_b200.model.unet.UNet, pdae_b200.model.shift_unet.ShiftUNet, pdae_b200.model.mlp_skip_net.MLPSkipNet,
    pdae_b200.model.representation_learning.{encoder,decoder,latent_denoise_fn}, pdae_b200.model.denoise_fn,
    pdae_b200.diffusion.gaussian_diffusion.GaussianDiffusion, pdae_b200.diffusion.ddim.DDIM
and ``pdae_b200.dropin.install()`` exposes them under the reference's import names (``model.*``,
``diffusion.*``) so its trainer/sampler scripts run unchanged.
"""
from .engine import get_default_precision, set_default_precision  # noqa: F401

__version__ = "0.1.0"
