"""Deterministic training on the GPU: under torch.use_deterministic_algorithms the PDAE step (semantic encoder + ShiftUNet), the
regular-DPM step (UNet with class labels and learned sigma) and their FusedAdamEMA updates give identical bits run after run,
in full precision, under bf16 autocast and with a GradScaler; their gradients match the default trainers' to within the
run-to-run spread; switching off returns to the default trainers."""
import copy
import warnings

import pytest
import torch

from pdae_b200.engine import DET_OPS, NONDET_OPS
from tests import cases
from tests.test_gpu_training_amp import AMP_SPREAD, FP32_SPREAD, _check_grads

pytestmark = pytest.mark.gpu
DEV = "cuda"
# 64-px ShiftUNet with attention at 16 x 16 (T = 256: the tensor-core attention backward under autocast)
SHIFT_CFG = dict(input_channel=3, base_channel=64, channel_multiplier=[1, 2, 2], num_residual_blocks_of_a_block=1,
                 attention_resolutions=[4], num_heads=1, head_channel=-1, use_new_attention_order=False, dropout=0.0,
                 latent_dim=512)
UNET_CFG = dict({k: v for k, v in SHIFT_CFG.items() if k != "latent_dim"}, num_class=5, learn_sigma=True)


@pytest.fixture(autouse=True)
def _deterministic():
    was, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn_only)


def _gd():
    from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
    return GaussianDiffusion(cases.DIFF, torch.device(DEV))


def _pdae_modules(size, dropout=0.0):
    from pdae_b200.model.representation_learning.encoder import CELEBA64Encoder, FFHQEncoder
    from pdae_b200.model.shift_unet import ShiftUNet
    from pdae_b200.utils.synth import fill_module_
    dec = fill_module_(ShiftUNet(**dict(SHIFT_CFG, dropout=dropout)), seed=6).to(DEV).train()
    dec.freeze()
    dec.set_train_mode()
    enc = fill_module_((CELEBA64Encoder if size == 64 else FFHQEncoder)(latent_dim=512), seed=7).to(DEV).train()
    dec.precision = enc.precision = "fp32"
    return [enc, dec]


def _unet_module(dropout=0.0):
    from pdae_b200.model.unet import UNet
    from pdae_b200.utils.synth import fill_module_
    net = fill_module_(UNet(**dict(UNET_CFG, dropout=dropout)), seed=5).to(DEV).train()
    net.precision = "fp32"
    return [net]


def _loss(kind, gd, mods, x0, cond):
    if kind == "pdae":
        return gd.representation_learning_train_one_batch(mods[0], mods[1], x0)["prediction_loss"]
    # regular_train_one_batch with a learned-sigma head: the eps half against the noise, a small term on the sigma half
    t = torch.randint(0, gd.timesteps, (x0.shape[0],), device=DEV, dtype=torch.long)
    noise = torch.randn_like(x0)
    out = mods[0](gd.q_sample(x_0=x0, t=t, noise=noise), t, cond)
    return gd.p_loss(noise, out[:, :3].contiguous()) + 1e-2 * out[:, 3:].square().mean()


def _run(kind, base, x0, cond=None, steps=3, amp=False, scaler=False, seed=0):
    """`steps` training steps (forward, backward, FusedAdamEMA.step) on deep copies of `base`: per step the loss and every
    gradient, then the parameters and the EMA parameters."""
    from pdae_b200.optim import FusedAdamEMA
    mods = [copy.deepcopy(m) for m in base]
    emas = [copy.deepcopy(m) for m in base]
    params = [p for m in mods for p in m.parameters() if p.requires_grad]
    opt = FusedAdamEMA(params, lr=1e-3, ema_decay=0.9)
    for m, e in zip(mods, emas):
        opt.attach_ema(m, e)
    sc = torch.amp.GradScaler("cuda") if scaler else None
    gd = _gd()
    torch.manual_seed(seed)
    out, ngrads = [], None
    for _ in range(steps):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            loss = _loss(kind, gd, mods, x0, cond)
        (sc.scale(loss) if sc else loss).backward()
        out.append(loss.detach().clone())
        grads = [p.grad.detach().clone() for p in params if p.grad is not None]
        ngrads = len(grads) if ngrads is None else ngrads
        out += grads
        if sc:
            sc.step(opt)
            sc.update()
        else:
            opt.step()
        opt.zero_grad(set_to_none=True)
    out += [p.detach().clone() for p in params]
    out += [p.detach().clone() for e in emas for p in e.parameters() if p.requires_grad]
    torch.cuda.synchronize()
    return out, mods, ngrads


def _inputs(kind, B, size):
    from pdae_b200.utils.synth import synth_images
    x0 = synth_images(B, 3, size, 31).to(DEV)
    cond = torch.arange(B, device=DEV) % UNET_CFG["num_class"] if kind == "unet" else None
    return x0, cond


def _trainers(mods):
    return [tr for m in mods for tr in m.__dict__.get("_train_cache", {}).values()]


def _plans(tr):
    return [p for p in (getattr(tr, "frozen", None), tr.fwd, tr.bwd) if p is not None]


MODES = [dict(amp=False), dict(amp=True), dict(amp=True, scaler=True)]
MODE_IDS = ["fp32", "bf16", "bf16-scaler"]
CASES = [("pdae", 64, 2, 0.1), ("pdae", 64, 4, 0.0), ("pdae", 128, 2, 0.0), ("unet", 64, 2, 0.1)]
CASE_IDS = ["pdae64-B2-dropout", "pdae64-B4", "pdae128-B2", "unet-classes-sigma-dropout"]


def _base(kind, size, dropout):
    return _pdae_modules(size, dropout) if kind == "pdae" else _unet_module(dropout)


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("kind,size,B,dropout", CASES, ids=CASE_IDS)
def test_training_steps_are_bitwise_reproducible(kind, size, B, dropout, mode):
    base = _base(kind, size, dropout)
    x0, cond = _inputs(kind, B, size)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        a, mods_a, _ = _run(kind, base, x0, cond, **mode)
        b, _, _ = _run(kind, base, x0, cond, **mode)          # fresh deep copies: freshly built trainers
    assert not [str(r.message) for r in w if "pdae_b200" in str(r.message)]
    assert len(a) == len(b)
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), f"tensor {i} of {len(a)} differs between two runs"
    assert all(torch.isfinite(t).all() for t in a)
    for tr in _trainers(mods_a):
        assert tr.det and tr.amp == mode["amp"]
        for P in _plans(tr):
            ops = {fn for fn, _ in P.ops}
            assert P.det and not ops & NONDET_OPS, sorted(ops & NONDET_OPS)
            assert {fn for fn in ops if fn.startswith(("conv_tc", "gemm_tc", "wgrad_tc"))} <= DET_OPS
            assert P._stats_elems == 0
    if kind == "pdae":
        bw = {fn for tr in _trainers(mods_a) for fn, _ in tr.bwd.ops}
        assert {"gn_bwd_sums_det", "gn_bwd_coef_det", "colsum_det", "conv2d_wgrad_simt_det"} <= bw
        assert ("wgrad_tc_bf16" if mode["amp"] else "wgrad_tc") in bw


@pytest.mark.parametrize("amp", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("kind,size,B,dropout", CASES[:1] + CASES[2:], ids=CASE_IDS[:1] + CASE_IDS[2:])
def test_deterministic_gradients_match_the_default_trainers(kind, size, B, dropout, amp):
    """One step with the switch on against the same step of the default (atomic) trainers."""
    base = _base(kind, size, dropout)
    x0, cond = _inputs(kind, B, size)
    det, _, n = _run(kind, base, x0, cond, steps=1, amp=amp)
    torch.use_deterministic_algorithms(False)
    ref, mods, _ = _run(kind, base, x0, cond, steps=1, amp=amp)
    assert not any(tr.det for tr in _trainers(mods))
    spread = AMP_SPREAD if amp else FP32_SPREAD
    loss_r = abs(float(det[0]) / float(ref[0]) - 1)
    print(f"{kind} {size}px amp={amp}: loss rel diff {loss_r:.2e}")
    assert loss_r <= (1e-3 if amp else 1e-5)
    _check_grads({str(i): g for i, g in enumerate(det[1:1 + n])}, {str(i): g for i, g in enumerate(ref[1:1 + n])},
                 f"deterministic vs default {kind} {size}px amp={amp}", **spread)


def test_switching_off_returns_to_the_default_trainers():
    base = _pdae_modules(64)
    x0, _ = _inputs("pdae", 2, 64)
    mods = [copy.deepcopy(m) for m in base]
    fresh = [copy.deepcopy(m) for m in base]
    gd = _gd()
    gd.representation_learning_train_one_batch(mods[0], mods[1], x0)["prediction_loss"].backward()
    torch.use_deterministic_algorithms(False)
    for ms in (mods, fresh):
        gd.representation_learning_train_one_batch(ms[0], ms[1], x0)["prediction_loss"].backward()
    for m, f in zip(mods, fresh):
        cache = m.__dict__["_train_cache"]
        assert len(cache) == 2 and sorted(tr.det for tr in cache.values()) == [False, True]
        plain = [tr for tr in cache.values() if not tr.det][0]
        ref = list(f.__dict__["_train_cache"].values())[0]
        for p, q in zip(_plans(plain), _plans(ref)):
            assert not p.det and [fn for fn, _ in p.ops] == [fn for fn, _ in q.ops]
    # the switch back on reuses the deterministic trainers
    torch.use_deterministic_algorithms(True, warn_only=True)
    gd.representation_learning_train_one_batch(mods[0], mods[1], x0)["prediction_loss"].backward()
    assert all(len(m.__dict__["_train_cache"]) == 2 for m in mods)
