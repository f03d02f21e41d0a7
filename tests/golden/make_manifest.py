#!/usr/bin/env python
"""Record state_dict key -> shape manifests of the REAL reference modules (run in the build container only)."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
REF = os.environ["PDAE_REFERENCE_DIR"]
sys.path.insert(0, REF)
import yaml  # noqa: E402
from model.unet import UNet  # noqa: E402
from model.shift_unet import ShiftUNet  # noqa: E402
from model.mlp_skip_net import MLPSkipNet  # noqa: E402
from model.representation_learning.encoder import CELEBA64Encoder, FFHQEncoder  # noqa: E402
from tests.configs import CELEBA64_PROXY, FFHQ128_PROXY, FFHQ_LATENT  # noqa: E402

mnist = yaml.load(open(os.path.join(REF, "config", "mnist_regular.yml")), Loader=yaml.FullLoader)["denoise_fn_config"]
mods = {
    "unet_mnist": (UNet(**mnist), mnist),
    "shiftunet_celeba64_proxy": (ShiftUNet(latent_dim=512, **CELEBA64_PROXY), dict(CELEBA64_PROXY, latent_dim=512)),
    "shiftunet_ffhq128_proxy": (ShiftUNet(latent_dim=512, **FFHQ128_PROXY), dict(FFHQ128_PROXY, latent_dim=512)),
    "encoder_celeba64": (CELEBA64Encoder(latent_dim=512), {"latent_dim": 512}),
    "encoder_ffhq": (FFHQEncoder(latent_dim=512), {"latent_dim": 512}),
    "mlp_ffhq_latent": (MLPSkipNet(**FFHQ_LATENT), FFHQ_LATENT),
}
out = {}
for name, (m, cfg) in mods.items():
    out[name] = {"cfg": cfg, "keys": {k: list(v.shape) for k, v in m.state_dict().items()},
                 "trainable": sorted(k for k, p in m.named_parameters() if p.requires_grad),
                 "zero_init": sorted(k for k, v in m.state_dict().items() if v.is_floating_point() and float(v.abs().max()) == 0.0)}
    print(name, len(out[name]["keys"]), "keys,", len(out[name]["trainable"]), "trainable,", len(out[name]["zero_init"]), "zero-init")
json.dump(out, open(os.path.join(HERE, "state_dict_manifest.json"), "w"), indent=0, sort_keys=True)
