"""Batch invariance under torch.use_deterministic_algorithms: an image's output bits depend on its own inputs, the weights, the
precision and its shape only -- not on the batch it is run in, its position there or the other images.

For every inference entry point and precision, a reference batch of N = 8 images is compared with torch.equal, image by
image, against each image run alone, the splits [3, 5] and [1, 7], the reversed batch, and the batch at offset 3 of a batch of
13 with five other images (13 % 2 and 13 % 8 leave partial two- and eight-image conv tiles at the 8 x 8 and 4 x 4 levels).
The 48-px cases have 24 x 24, 12 x 12 and 6 x 6 levels, whose conv tiles hold parts of several images.  The sharded
autoencoding is emulated rank by rank for world sizes 1-4.  With the switch off one case is held to the default plans'
golden tolerances."""
import pytest
import torch

from tests import cases
from tests.configs import FFHQ_LATENT
from tests.test_gpu_parity import check
from tests.util import load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
PRECISIONS = ["fp32", "bf16", "bf16x3"]
N = 8                 # the reference batch: pool images 0..7; pool images 8..12 are the others
# three levels (S, S/2, S/4) with attention at S/2
SHIFT = dict(load_golden("model_shiftunet_b64")[0]["cfg"], channel_multiplier=[1, 2, 2], num_residual_blocks_of_a_block=1)
UNET = dict({k: v for k, v in SHIFT.items() if k != "latent_dim"}, num_class=10)
FFHQ = {k: v for k, v in FFHQ_LATENT.items() if k != "model"}
BATCHES = ([[i] for i in range(N)] + [[0, 1, 2], [3, 4, 5, 6, 7], list(range(1, N)), list(range(N - 1, -1, -1)),
                                      [8, 9, 10] + list(range(N)) + [11, 12]])


@pytest.fixture(autouse=True)
def deterministic():
    was, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn_only)


def _module(kind, precision):
    from pdae_b200.model.mlp_skip_net import MLPSkipNet
    from pdae_b200.model.representation_learning.encoder import CELEBA64Encoder, FFHQEncoder
    from pdae_b200.model.shift_unet import ShiftUNet
    from pdae_b200.model.unet import UNet
    from pdae_b200.utils.synth import fill_module_
    m = {"shift": lambda: ShiftUNet(**SHIFT), "unet": lambda: UNet(**UNET), "enc64": lambda: CELEBA64Encoder(latent_dim=512),
         "enc128": lambda: FFHQEncoder(latent_dim=512), "mlp": lambda: MLPSkipNet(**FFHQ)}[kind]()
    m = fill_module_(m, seed=61).eval().to(DEV)
    m.precision = precision
    return m


def _pool(seed, size=None):
    """Per-image inputs of the 13 pool images: x (or z_t), t, z, class labels and a second image / latent."""
    from pdae_b200.utils.synth import synth_images, synth_normal
    n = N + 5
    p = {"t": torch.arange(n, dtype=torch.int64, device=DEV) * 73 % 1000,
         "label": torch.arange(n, dtype=torch.int64, device=DEV) % 10,
         "z": synth_normal((n, 512), seed + 1).to(DEV), "z2": synth_normal((n, 512), seed + 2).to(DEV)}
    if size is not None:
        p["x"] = synth_images(n, 3, size, seed).to(DEV)
        p["y"] = synth_images(n, 3, size, seed + 3).to(DEV)
    return p


def _outputs(o):
    return tuple(o) if isinstance(o, (tuple, list)) else (o,)


def _check(run, pool, what):
    """run(inputs) -> output tensor(s) with the batch first; inputs = the pool entries of one batch."""
    def call(idx):
        ix = torch.tensor(idx, device=DEV)
        with torch.no_grad():
            return _outputs(run({k: v[ix] for k, v in pool.items()}))
    ref = call(list(range(N)))
    for idx in BATCHES:
        out = call(idx)
        for k, i in enumerate(idx):
            if i >= N:
                continue
            for j, (o, r) in enumerate(zip(out, ref)):
                assert torch.equal(o[k], r[i]), (f"{what}: image {i} at position {k} of a batch of {len(idx)} (output {j}): "
                                                 f"max |d| = {float((o[k] - r[i]).abs().max()):.3e}")


def _gd():
    from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
    return GaussianDiffusion(cases.DIFF, DEV)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("size", [16, 48])
def test_unet_with_class_labels(size, precision):
    m = _module("unet", precision)
    _check(lambda p: m(p["x"], p["t"], p["label"]), _pool(1, size), f"UNet {size}px {precision}")


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("size", [16, 48])
def test_shiftunet(size, precision):
    m = _module("shift", precision)
    _check(lambda p: m(p["x"], p["t"], p["z"]), _pool(2, size), f"ShiftUNet {size}px {precision}")


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("kind", ["enc64", "enc128"])
def test_encoders(kind, precision):
    m = _module(kind, precision)
    _check(lambda p: m(p["x"]), _pool(3, 64 if kind == "enc64" else 128), f"{kind} {precision}")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_mlp_skip_net_and_latent_loop(precision):
    from pdae_b200.diffusion.ddim import DDIM
    m = _module("mlp", precision)
    _check(lambda p: m(p["z"], p["t"]), _pool(4), f"MLPSkipNet {precision}")
    d = _gd()
    nb, tmap = d.get_ddim_betas_and_timestep_map("ddim10", d.latent_diffusion_config["alphas_cumprod"].cpu().numpy())
    dd = DDIM(nb, tmap, DEV)
    _check(lambda p: dd.latent_ddim_sample_loop(m, p["z"]), _pool(5), f"latent ddim10 loop {precision}")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_ddim_loops(precision):
    unet, shift = _module("unet", precision), _module("shift", precision)
    dd = _gd()._ddim("ddim4")
    pool = _pool(6, 16)
    _check(lambda p: dd.ddim_sample_loop(unet, p["x"], p["label"]), pool, f"ddim_sample_loop {precision}")
    _check(lambda p: dd.ddim_encode_loop(unet, p["x"], p["label"]), pool, f"ddim_encode_loop {precision}")
    _check(lambda p: dd.shift_ddim_sample_loop(shift, p["z"], p["x"], stop_percent=0.5), pool,
           f"shift_ddim_sample_loop(stop_percent=0.5) {precision}")
    _check(lambda p: dd.shift_ddim_trajectory_interpolation(shift, p["z"], p["z2"], p["x"], 0.3), pool,
           f"trajectory interpolation {precision}")
    _check(lambda p: dd.shift_ddim_sample_loop(shift, p["z"], p["x"], stop_percent=0.5), _pool(7, 48),
           f"shift_ddim_sample_loop 48px {precision}")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_autoencoding_and_its_shards(precision):
    from pdae_b200.utils.dist import shard_range
    enc, dec = _module("enc64", precision), _module("shift", precision)
    gd = _gd()

    def auto(x):
        return gd.representation_learning_autoencoding("ddim3", "ddim3", enc, dec, x)
    pool = _pool(8, 64)
    _check(lambda p: auto(p["x"]), pool, f"representation_learning_autoencoding {precision}")
    x = pool["x"][:N]
    with torch.no_grad():
        whole = auto(x)
        for world in range(1, 5):
            # what sharded_autoencode runs on each rank, gathered in rank order
            parts = [auto(x[s:e]) for s, e in (shard_range(N, r, world) for r in range(world)) if e > s]
            assert torch.equal(torch.cat(parts), whole), f"sharded autoencoding, world size {world}, {precision}"


def test_metrics():
    from pdae_b200.metric import utils as metric
    for size in (16, 48):
        pool = _pool(9, size)
        _check(lambda p: metric.calculate_mse(p["x"], p["y"]), pool, f"calculate_mse {size}px")
        _check(lambda p: metric.calculate_ssim(p["x"], p["y"]), pool, f"calculate_ssim {size}px")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_tensor_core_slots_are_per_image(precision):
    """Every DET tensor-core op of a deterministic plan sizes its slots per image: the workspace at B is B times that at 1."""
    for kind, size in (("shift", 48), ("shift", 16), ("enc64", 64)):
        m = _module(kind, precision)
        p = _pool(10, size)
        sizes = {}
        for B in (1, 13):
            with torch.no_grad():
                m(p["x"][:B]) if kind == "enc64" else m(p["x"][:B], p["t"][:B], p["z"][:B])
            plan = [pl for (k, _, det), (pl, _) in m._plans().items() if det and k[1] == B][0]
            sizes[B] = [int(q(h)) for _, _, q, h in plan._det_handles]
        assert sizes[13] == [13 * n for n in sizes[1]], (kind, size, precision, sizes)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_switch_off_keeps_the_default_plans_within_tolerance(precision):
    m = _module("shift", precision)
    p = _pool(11, 48)
    with torch.no_grad():
        det = m(p["x"][:N], p["t"][:N], p["z"][:N])
        torch.use_deterministic_algorithms(False)
        ref = m(p["x"][:N], p["t"][:N], p["z"][:N])
    assert not any(pl.det for (_, _, d), (pl, _) in m._plans().items() if not d)
    check(det[0], ref[0], precision, f"48px eps, deterministic vs default ({precision})")
    check(det[1], ref[1], precision, f"48px shift, deterministic vs default ({precision})")
