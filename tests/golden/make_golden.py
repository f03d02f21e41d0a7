#!/usr/bin/env python
"""Generate tests/golden/*.npz by running the REAL reference (ckczzj/PDAE, sources at $PDAE_REFERENCE_DIR).

Run only where the reference sources are available:
    python tests/golden/make_golden.py
Each fixture stores the config (JSON), the input seeds and the reference outputs.  Weights are NOT
stored: both sides regenerate them with pdae_b200.utils.synth (numpy PCG64 keyed by parameter
name), so a fixture is a few KB.  The oracle (oracle/pdae_oracle.py) and the CUDA path are both
checked against these files.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ["PDAE_REFERENCE_DIR"])

from pdae_b200.utils.synth import fill_module_, synth_images, synth_normal  # noqa: E402

import model.module as rm  # noqa: E402  (reference)
from model.unet import UNet  # noqa: E402
from model.shift_unet import ShiftUNet  # noqa: E402
from model.mlp_skip_net import MLPSkipNet  # noqa: E402
from model.representation_learning.encoder import CELEBA64Encoder, FFHQEncoder  # noqa: E402
from diffusion.gaussian_diffusion import GaussianDiffusion  # noqa: E402
from diffusion.ddim import DDIM  # noqa: E402

torch.set_grad_enabled(False)
torch.set_num_threads(8)

TINY_UNET = dict(input_channel=3, base_channel=32, channel_multiplier=[1, 2, 2],
                 num_residual_blocks_of_a_block=1, attention_resolutions=[2], num_heads=1, head_channel=-1,
                 use_new_attention_order=False, dropout=0.0)
TINY_UNET_NEW = dict(TINY_UNET, use_new_attention_order=True, num_heads=2, attention_resolutions=[2, 4])
TINY_UNET_HC = dict(TINY_UNET, head_channel=32, learn_sigma=True)
TINY_UNET_CLS = dict(TINY_UNET, num_class=10, input_channel=1, attention_resolutions=[])
TINY_SHIFT = dict(TINY_UNET, latent_dim=64)
TINY_SHIFT2 = dict(input_channel=3, base_channel=64, channel_multiplier=[1, 2], num_residual_blocks_of_a_block=2,
                   attention_resolutions=[2], num_heads=1, head_channel=-1, use_new_attention_order=False,
                   dropout=0.0, latent_dim=512)
TINY_MLP = dict(input_channel=64, model_channel=128, num_layers=4, time_emb_channel=32, use_norm=True, dropout=0.0)
DIFF = {"timesteps": 1000, "betas_type": "linear"}


def save(name, cfg, **arrays):
    out = {k: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in arrays.items()}
    np.savez_compressed(os.path.join(HERE, name + ".npz"), cfg=np.array(json.dumps(cfg)), **out)
    print("wrote", name, {k: v.shape for k, v in out.items()})


def block_cases():
    B, E = 2, 128
    emb = synth_normal((B, E), 11)
    embz = synth_normal((B, E), 12)
    for name, kw, shift in [
        ("res_same", dict(channels=64), False), ("res_widen", dict(channels=32, out_channels=64), False),
        ("res_narrow", dict(channels=96, out_channels=32), False), ("res_up", dict(channels=32, up=True), False),
        ("res_down", dict(channels=32, down=True), False), ("shift_same", dict(channels=64), True),
        ("shift_narrow", dict(channels=96, out_channels=32), True), ("shift_up", dict(channels=32, up=True), True),
    ]:
        cls = rm.ResBlockShift if shift else rm.ResBlock
        m = fill_module_(cls(emb_channels=E, dropout=0.0, **kw), seed=3).eval()
        x = synth_normal((B, kw["channels"], 8, 8), 13)
        y = m(x, emb, embz) if shift else m(x, emb)
        save("block_" + name, dict(kind="resblock", shift=shift, emb_channels=E, **kw), y=y)
    for name, C, heads, new in [("attn_legacy_h1", 64, 1, False), ("attn_legacy_h4", 128, 4, False),
                                ("attn_new_h1", 64, 1, True), ("attn_new_h4", 128, 4, True)]:
        m = fill_module_(rm.AttentionBlock(C, heads, -1, new), seed=4).eval()
        x = synth_normal((B, C, 8, 8), 14)
        save("block_" + name, dict(kind="attention", channels=C, heads=heads, new_order=new), y=m(x))
    t = torch.tensor([0, 1, 17, 999], dtype=torch.long)
    save("timestep_embedding", dict(kind="temb"), t=t, e64=rm.timestep_embedding(t, 64), e33=rm.timestep_embedding(t, 33))


def model_cases():
    t = torch.tensor([3, 977], dtype=torch.long)
    for name, cfg, size in [("unet_tiny", TINY_UNET, 16), ("unet_new_order", TINY_UNET_NEW, 16),
                            ("unet_headch_sigma", TINY_UNET_HC, 16)]:
        m = fill_module_(UNet(**cfg), seed=5).eval()
        x = synth_normal((2, cfg["input_channel"], size, size), 15)
        save("model_" + name, dict(kind="unet", cfg=cfg, size=size), t=t, y=m(x, t))
    m = fill_module_(UNet(**TINY_UNET_CLS), seed=5).eval()
    x = synth_normal((2, 1, 32, 32), 15)
    cond = torch.tensor([1, 7], dtype=torch.long)
    save("model_unet_class", dict(kind="unet", cfg=TINY_UNET_CLS, size=32), t=t, cond=cond, y=m(x, t, cond))
    for name, cfg, size in [("shiftunet_tiny", TINY_SHIFT, 16), ("shiftunet_b64", TINY_SHIFT2, 16)]:
        m = fill_module_(ShiftUNet(**cfg), seed=6).eval()
        x = synth_normal((2, 3, size, size), 16)
        z = synth_normal((2, cfg["latent_dim"]), 17)
        eps, grad = m(x, t, z)
        save("model_" + name, dict(kind="shiftunet", cfg=cfg, size=size), t=t, eps=eps, grad=grad)
    for name, cls, size in [("encoder_celeba64", CELEBA64Encoder, 64), ("encoder_ffhq128", FFHQEncoder, 128)]:
        m = fill_module_(cls(latent_dim=512), seed=7).eval()
        save("model_" + name, dict(kind="encoder", size=size), z=m(synth_images(2, 3, size, 18)))
    m = fill_module_(MLPSkipNet(**TINY_MLP), seed=8).eval()
    save("model_mlp_skip", dict(kind="mlp", cfg=TINY_MLP), t=t, y=m(synth_normal((2, 64), 19), t))


def diffusion_cases():
    for bt in ("linear", "cosine"):
        gd = GaussianDiffusion({"timesteps": 1000, "betas_type": bt}, "cpu")
        tabs = {k: v for k, v in vars(gd).items() if isinstance(v, torch.Tensor)}
        save("diffusion_tables_" + bt, dict(kind="tables", betas_type=bt), **tabs)
    gd = GaussianDiffusion(DIFF, "cpu")
    arrs = {}
    for style in ("ddim10", "ddim100", "ddim200", "ddim500", "ddim1000"):
        nb, tmap = gd.get_ddim_betas_and_timestep_map(style, gd.alphas_cumprod.cpu().numpy())
        arrs[style + "_betas"] = nb
        arrs[style + "_map"] = tmap
        if style in ("ddim10", "ddim100"):
            d = DDIM(nb, tmap, "cpu")
            for k, v in vars(d).items():
                if isinstance(v, torch.Tensor) and k != "timestep_map":
                    arrs[f"{style}_{k}"] = v
    save("diffusion_ddim_maps", dict(kind="ddim_maps"), **arrs)

    # elementwise steps
    x0 = synth_images(4, 3, 8, 21)
    noise = synth_normal((4, 3, 8, 8), 22)
    t = torch.tensor([0, 1, 500, 999], dtype=torch.long)
    torch.manual_seed(1234)
    eps = synth_normal((4, 3, 8, 8), 23)
    ps = gd.noise_p_sample(x0, t, eps)          # draws torch.randn(shape) internally
    torch.manual_seed(1234)
    ps_noise = torch.randn(x0.shape)
    lr = synth_normal((4, 3, 8, 8), 24).clamp(-1, 1)
    torch.manual_seed(1234)
    ps_lr = gd.noise_p_sample(x0, t, eps, lr)
    save("diffusion_steps", dict(kind="steps"), t=t, q=gd.q_sample(x0, t, noise), p_sample=ps, p_noise=ps_noise,
         p_sample_lr=ps_lr)

    # loops on tiny nets
    unet = fill_module_(UNet(**TINY_UNET), seed=5).eval()
    xT = synth_normal((2, 3, 16, 16), 25)
    x0 = synth_images(2, 3, 16, 26)
    save("loop_unet_ddim10", dict(kind="loop_unet", cfg=TINY_UNET, size=16),
         sample=gd.ddim_sample("ddim10", unet, xT), encode=gd.ddim_encode("ddim10", unet, x0))
    dec = fill_module_(ShiftUNet(**TINY_SHIFT), seed=6).eval()
    z = synth_normal((2, 64), 27)
    save("loop_shift_ddim10", dict(kind="loop_shift", cfg=TINY_SHIFT, size=16),
         sample=gd.representation_learning_ddim_sample("ddim10", None, dec, None, xT, z),
         sample_stop30=gd.representation_learning_ddim_sample("ddim10", None, dec, None, xT, z, stop_percent=0.3),
         encode=gd.representation_learning_ddim_encode("ddim10", None, dec, x0, z))

    # full autoencoding with a real encoder (64 px) -- the benchmark workload in miniature
    cfg = dict(TINY_SHIFT, latent_dim=512)
    dec = fill_module_(ShiftUNet(**cfg), seed=6).eval()
    enc = fill_module_(CELEBA64Encoder(latent_dim=512), seed=7).eval()
    x0 = synth_images(2, 3, 64, 28)
    save("loop_autoencode_ddim10", dict(kind="autoencode", cfg=cfg, size=64),
         recon=gd.representation_learning_autoencoding("ddim10", "ddim10", enc, dec, x0))

    # latent sampling loop
    mlp = fill_module_(MLPSkipNet(**TINY_MLP), seed=8).eval()
    lat = gd.latent_diffusion_config["alphas_cumprod"]
    nb, tmap = gd.get_ddim_betas_and_timestep_map("ddim10", lat.cpu().numpy())
    zT = synth_normal((2, 64), 29).clamp(-1, 1)
    save("loop_latent_ddim10", dict(kind="latent_loop", cfg=TINY_MLP), z=DDIM(nb, tmap, "cpu").latent_ddim_sample_loop(mlp, zT))


def glue_cases():
    """The thin wrappers around the hot path (SURVEY.md section 8 rows a20, a22, a24): trajectory interpolation, the x_0-clip
    ancestral step, the DDPM loops, latent sampling with stop_percent=0.3, manipulation, gap measure, one-step denoising.
    Every random draw of the reference comes from the default CPU generator after torch.manual_seed(seed): the tests replay
    the same stream through GaussianDiffusion._randn / _randn_like / _rand_like."""
    gd = GaussianDiffusion(DIFF, "cpu")
    dec16 = fill_module_(ShiftUNet(**TINY_SHIFT), seed=6).eval()
    xT = synth_normal((2, 3, 16, 16), 25)
    z1, z2 = synth_normal((2, 64), 27), synth_normal((2, 64), 61)
    save("glue_interpolation", dict(kind="glue_interp", cfg=TINY_SHIFT, size=16, alpha=0.3, style="ddim10"),
         y=gd.representation_learning_ddim_trajectory_interpolation("ddim10", dec16, z1, z2, xT, 0.3))

    # x_0_clip_p_sample (gaussian_diffusion.py:130-146): fixed + learned variance, with / without the clip
    x_t = synth_normal((4, 3, 8, 8), 62)
    eps = synth_normal((4, 3, 8, 8), 63)
    lr = synth_normal((4, 3, 8, 8), 64).clamp(-1, 1)
    t = torch.tensor([0, 1, 500, 999], dtype=torch.long)
    out = {}
    for name, kw in (("fixed_clip", {}), ("fixed_noclip", dict(clip_x_0=False)), ("learned_clip", dict(learned_range=lr))):
        torch.manual_seed(4321)
        out[name] = gd.x_0_clip_p_sample(x_t.clone(), t, eps, **kw)
    save("glue_x0_clip", dict(kind="glue_x0_clip", seed=4321), t=t, **out)

    # DDPM ancestral loops on a short schedule (T=20): plain UNet, learn_sigma UNet, ShiftUNet
    gd20 = GaussianDiffusion({"timesteps": 20, "betas_type": "linear"}, "cpu")
    unet = fill_module_(UNet(**TINY_UNET), seed=5).eval()
    unet_ls = fill_module_(UNet(**TINY_UNET_HC), seed=5).eval()
    torch.manual_seed(555)
    y_reg = gd20.regular_ddpm_sample(unet, xT)
    torch.manual_seed(556)
    y_ls = gd20.regular_ddpm_sample(unet_ls, xT)
    z = synth_normal((2, 64), 27)
    torch.manual_seed(557)
    y_rl = gd20.representation_learning_ddpm_sample(None, dec16, xT, xT, z)
    save("glue_ddpm", dict(kind="glue_ddpm", timesteps=20, cfg_unet=TINY_UNET, cfg_sigma=TINY_UNET_HC, cfg_shift=TINY_SHIFT,
                           size=16, seeds=[555, 556, 557]), regular=y_reg, learned_sigma=y_ls, representation=y_rl)

    # latent_diffusion_sample (:400-415): draws z_T inside, clamps it, latent DDIM loop, decoder loop with stop_percent=0.3
    mlp = fill_module_(MLPSkipNet(**TINY_MLP), seed=8).eval()
    mean, std = synth_normal((1, 64), 65) * 0.1, synth_normal((1, 64), 66).abs() + 0.5
    torch.manual_seed(558)
    y = gd.latent_diffusion_sample("ddim10", "ddim10", mlp, dec16, xT, mean, std)
    save("glue_latent_sample", dict(kind="glue_latent_sample", cfg_mlp=TINY_MLP, cfg_shift=TINY_SHIFT, size=16, seed=558), y=y)

    # manipulation_sample (:435-443), gap measure (:292-318) and one-step denoising (:320-334) on the 64-px tiny autoencoder
    cfg = dict(TINY_SHIFT, latent_dim=512)
    dec = fill_module_(ShiftUNet(**cfg), seed=6).eval()
    enc = fill_module_(CELEBA64Encoder(latent_dim=512), seed=7).eval()
    x0 = synth_images(2, 3, 64, 28)
    xT64 = synth_normal((2, 3, 64, 64), 67)
    mean, std = synth_normal((1, 512), 34) * 0.1, synth_normal((1, 512), 35).abs() + 0.5
    cw = synth_normal((5, 512), 68)
    save("glue_manipulation", dict(kind="glue_manipulation", cfg=cfg, size=64, class_id=3, scale=0.3, style="ddim10"),
         y=gd.manipulation_sample("ddim10", cw, enc, dec, x0, xT64, mean, std, 3, 0.3))
    gd8 = GaussianDiffusion({"timesteps": 8, "betas_type": "linear"}, "cpu")
    torch.manual_seed(559)
    gp, ga = gd8.representation_learning_gap_measure(enc, dec, x0)
    save("glue_gap", dict(kind="glue_gap", cfg=cfg, size=64, timesteps=8, seed=559), gap_pred=np.array(gp), gap_ae=np.array(ga))
    torch.manual_seed(560)
    p0, a0 = gd.representation_learning_denoise_one_step(enc, dec, x0, [10, 700])
    save("glue_denoise_one_step", dict(kind="glue_denoise", cfg=cfg, size=64, seed=560, timesteps=[10, 700]), pred=p0, ae=a0)


def training_cases():
    torch.set_grad_enabled(True)
    gd = GaussianDiffusion(DIFF, "cpu")
    cfg = dict(TINY_SHIFT, latent_dim=512)
    dec = fill_module_(ShiftUNet(**cfg), seed=6)
    enc = fill_module_(CELEBA64Encoder(latent_dim=512), seed=7)
    x0 = synth_images(2, 3, 64, 31)
    torch.manual_seed(777)
    loss = gd.representation_learning_train_one_batch(enc, dec, x0)["prediction_loss"]
    loss.backward()
    torch.manual_seed(777)
    t = torch.randint(0, 1000, (2,), dtype=torch.long)
    noise = torch.randn_like(x0)
    grads = {"g_" + k.replace(".", "_"): p.grad for k, p in list(dec.named_parameters()) + [("enc." + k, p) for k, p in enc.named_parameters()]
             if p.grad is not None and k.endswith(("label_emb.weight", "shift_out.2.weight", "shift_middle_block.0.in_layers.2.weight",
                                                    "shift_output_blocks.0.0.emb_z_layers.1.weight", "encoder.0.weight", "encoder.14.weight"))}
    n_grad = sum(1 for p in list(dec.parameters()) + list(enc.parameters()) if p.grad is not None)
    save("train_representation_learning", dict(kind="train_rl", cfg=cfg, size=64, n_params_with_grad=n_grad),
         t=t, noise=noise, loss=loss.detach(),
         **{k: v.detach().flatten()[:512] for k, v in grads.items()},
         **{"n" + k: v.detach().double().norm().float() for k, v in grads.items()})
    unet = fill_module_(UNet(**TINY_UNET), seed=5)
    x0 = synth_images(2, 3, 16, 32)
    torch.manual_seed(778)
    loss = gd.regular_train_one_batch(unet, x0)["prediction_loss"]
    torch.manual_seed(778)
    t = torch.randint(0, 1000, (2,), dtype=torch.long)
    noise = torch.randn_like(x0)
    save("train_regular", dict(kind="train_regular", cfg=TINY_UNET, size=16), t=t, noise=noise, loss=loss.detach())
    latent_training_case(gd)
    torch.set_grad_enabled(False)


def latent_training_case(gd):
    """latent_diffusion_train_one_batch (gaussian_diffusion.py:373-398): frozen encoder, trainable MLPSkipNet, L1 loss."""
    cfg = dict(TINY_MLP, input_channel=512, model_channel=256, num_layers=5)
    mlp = fill_module_(MLPSkipNet(**cfg), seed=9)
    enc = fill_module_(CELEBA64Encoder(latent_dim=512), seed=7).requires_grad_(False).eval()
    x0 = synth_images(3, 3, 64, 33)
    mean, std = synth_normal((1, 512), 34) * 0.1, synth_normal((1, 512), 35).abs() + 0.5
    torch.manual_seed(779)
    loss = gd.latent_diffusion_train_one_batch(mlp, enc, x0, mean, std)["prediction_loss"]
    loss.backward()
    with torch.no_grad():
        z0 = gd.normalize(enc(x0), mean, std)
    torch.manual_seed(779)
    t = torch.randint(0, 1000, (3,), dtype=torch.long)
    noise = torch.randn_like(z0)
    keys = ("time_embed.0.weight", "time_embed.2.bias", "layers.0.linear.weight", "layers.1.linear_emb.weight",
            "layers.2.norm.weight", "layers.3.norm.bias", "layers.4.linear.weight", "layers.4.linear.bias")
    grads = {k: p.grad for k, p in mlp.named_parameters() if k in keys}
    assert len(grads) == len(keys)
    n_grad = sum(1 for p in mlp.parameters() if p.grad is not None)
    save("train_latent", dict(kind="train_latent", cfg=cfg, n_params_with_grad=n_grad), t=t, noise=noise, z0=z0,
         loss=loss.detach(), **{"g_" + k.replace(".", "_"): v.flatten()[:512] for k, v in grads.items()},
         **{"n_" + k.replace(".", "_"): v.double().norm().float() for k, v in grads.items()})


def caller_cases():
    """SURVEY.md §8(f) rows: optimizer + EMA, wire formats, metrics -- the callers either side of the hot path."""
    from metric.utils import calculate_mse, calculate_ssim  # noqa: E402 (reference; imports torch + PIL only)
    import torchvision.transforms as T
    a = synth_images(3, 3, 40, 41)
    b = (a + 0.1 * synth_normal((3, 3, 40, 40), 42)).clamp(-1, 1)
    # the trainers' / samplers' image conversion, trainer/train_representation_learning.py:173-174 (expression as used there)
    u8 = (b * 1.3).mul(0.5).add(0.5).mul(255).add(0.5).clamp(0, 255).permute(0, 2, 3, 1).to("cpu", torch.uint8)
    # dataset/ffhq.py:27-31 (no Resize: the fixture is already at size): ToTensor + Normalize on each HWC uint8 image
    tf = T.Compose([T.ToTensor(), T.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))])
    back = torch.stack([tf(img.numpy()) for img in u8])
    save("caller_metrics_io", dict(kind="caller_io", n=3, size=40), mse=calculate_mse(a, b), ssim=calculate_ssim(a, b),
         u8=u8, back=back)
    # Adam exactly as trainer/train_representation_learning.py:57-69 builds it (config/ffhq_representation_learning.yml:33-37)
    # and the EMA loop of :192-212 with ema_every=1, ema_decay=0.9999 (:46-47)
    torch.set_grad_enabled(True)
    shapes = [(64, 3, 3, 3), (64,), (37,), (128, 64), (5, 7, 3)]
    ps = [torch.nn.Parameter(synth_normal(s, 50 + i) * 0.1) for i, s in enumerate(shapes)]
    ema = [p.detach().clone() for p in ps]
    opt = torch.optim.Adam([{"params": ps[:2]}, {"params": ps[2:]}], lr=float("1e-4"), betas=eval("(0.9, 0.999)"),
                           eps=float("1e-8"), weight_decay=float("0.0"))
    for step in range(4):
        for i, p in enumerate(ps):
            p.grad = synth_normal(tuple(p.shape), 100 + 10 * step + i) * (10.0 ** (i - 2))
        opt.step()
        for e, p in zip(ema, ps):
            e.data.mul_(0.9999).add_(p.data, alpha=1.0 - 0.9999)
    torch.set_grad_enabled(False)
    save("caller_adam_ema", dict(kind="caller_adam", shapes=shapes, steps=4, lr=1e-4, betas=[0.9, 0.999], eps=1e-8,
                                 weight_decay=0.0, ema_decay=0.9999),
         **{f"p{i}": p.detach() for i, p in enumerate(ps)}, **{f"e{i}": e for i, e in enumerate(ema)})
    # weight decay + a larger lr so every term of the update is exercised
    ps = [torch.nn.Parameter(synth_normal(s, 50 + i) * 0.1) for i, s in enumerate(shapes)]
    opt = torch.optim.Adam(ps, lr=3e-3, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.01)
    torch.set_grad_enabled(True)
    for step in range(3):
        for i, p in enumerate(ps):
            p.grad = synth_normal(tuple(p.shape), 100 + 10 * step + i)
        opt.step()
    torch.set_grad_enabled(False)
    save("caller_adam_wd", dict(kind="caller_adam", shapes=shapes, steps=3, lr=3e-3, betas=[0.8, 0.95], eps=1e-6,
                                weight_decay=0.01, ema_decay=-1.0), **{f"p{i}": p.detach() for i, p in enumerate(ps)})


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "glue":      # regenerate only the round-2 glue fixtures
        glue_cases()
        sys.exit(0)
    block_cases()
    model_cases()
    diffusion_cases()
    glue_cases()
    training_cases()
    caller_cases()
