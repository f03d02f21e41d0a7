"""CUDA path vs the fixtures recorded from the real reference and vs the CPU oracle (same seeded inputs).

fp32 mode and the split-operand tensor-core mode "bf16x3": rtol 1e-3 / atol 1e-4 (BASELINE.json north_star).  bf16 tensor-core mode (stated tolerance): relative L2
error <= 2e-2 and elementwise |err| <= 5e-2 * max|ref| -- bf16 operands carry 8 mantissa bits; accumulation, GroupNorm
statistics, the residual stream and the DDIM update stay fp32."""
import pytest
import torch

from oracle import pdae_oracle as O
from tests import cases
from tests.util import assert_close, golden_names, load_golden, rel_l2

pytestmark = pytest.mark.gpu

FP32 = dict(rtol=1e-3, atol=1e-4)


def check(got, want, precision, what):
    if precision in ("fp32", "bf16x3"):   # the split-operand tensor-core mode is held to the fp32 tolerance
        if precision == "bf16x3":
            print(f"[bf16x3] {what}: rel-L2 {rel_l2(got, want):.3e}")
        assert_close(got, want, what=what, **FP32)
    else:
        r = rel_l2(got, want)
        print(f"[bf16] {what}: rel-L2 {r:.3e}")
        assert r <= 2e-2, f"{what}: bf16 rel-L2 {r:.3e} > 2e-2"
        assert_close(got, want, rtol=0.0, atol=5e-2 * float(want.abs().max()), what=what + " (bf16)")


def _cuda(d):
    return {k: v.cuda() for k, v in d.items()}


@pytest.mark.parametrize("precision", ["fp32", "bf16", "bf16x3"])
@pytest.mark.parametrize("name", golden_names("block_"))
def test_blocks(name, precision):
    cfg, g = load_golden(name)
    m, inp = cases.block_case(cfg)
    m = m.cuda()
    m.precision = precision
    i = _cuda(inp)
    with torch.no_grad():
        y = m(i["x"], i["emb"], i["emb_z"]) if "emb_z" in i else (m(i["x"], i["emb"]) if "emb" in i else m(i["x"]))
    check(y, g["y"], precision, name)


def test_timestep_embedding():
    from pdae_b200.model.module import timestep_embedding
    _, g = load_golden("timestep_embedding")
    assert_close(timestep_embedding(g["t"].cuda(), 64), g["e64"], rtol=1e-6, atol=2e-6, what="e64")
    assert_close(timestep_embedding(g["t"].cuda(), 33), g["e33"], rtol=1e-6, atol=2e-6, what="e33")


@pytest.mark.parametrize("precision", ["fp32", "bf16", "bf16x3"])
@pytest.mark.parametrize("name", golden_names("model_"))
def test_models(name, precision):
    cfg, g = load_golden(name)
    m, inp = cases.model_case(cfg)
    m = m.cuda()
    m.precision = precision
    i = _cuda(inp)
    with torch.no_grad():
        if cfg["kind"] == "unet":
            check(m(i["x"], g["t"].cuda(), g["cond"].cuda() if "cond" in g else None), g["y"], precision, name)
        elif cfg["kind"] == "shiftunet":
            eps, grad = m(i["x"], g["t"].cuda(), i["z"])
            check(eps, g["eps"], precision, name + ".eps")
            check(grad, g["grad"], precision, name + ".grad")
        elif cfg["kind"] == "encoder":
            check(m(i["x"]), g["z"], precision, name)
        else:
            check(m(i["x"], g["t"].cuda()), g["y"], precision, name)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_repeat_calls_and_weight_update_refresh_packed_weights(precision):
    """Plans cache packed weights; an in-place parameter update (optimizer step / load_state_dict) must be seen -- in every
    mode (each packs differently: fp32 tap-major, bf16 K-major, bf16x3 [W_hi | W_hi | W_lo], the fused skip / head variants)."""
    cfg, g = load_golden("model_shiftunet_b64")
    m, inp = cases.model_case(cfg)
    m = m.cuda()
    m.precision = precision
    i = _cuda(inp)
    t = g["t"].cuda()
    with torch.no_grad():
        e1, g1 = m(i["x"], t, i["z"])
        e2, g2 = m(i["x"], t, i["z"])
        # GroupNorm statistics are accumulated with atomics -> run-to-run differences at the 1e-7 level are expected
        # (1e-5 in the split-operand mode, where a last-bit change can move a value across a bf16 hi/lo boundary)
        rep = dict(rtol=1e-3, atol=1e-4) if precision == "bf16x3" else dict(rtol=1e-4, atol=1e-5)
        assert_close(e2, e1, what="repeat eps", **rep)
        assert_close(g2, g1, what="repeat grad", **rep)
        sd = {k: v.clone() for k, v in m.state_dict().items()}
        m.shift_out[2].weight.mul_(2.0)
        m.shift_out[2].bias.mul_(2.0)
        _, g3 = m(i["x"], t, i["z"])
        tol = dict(rtol=1e-4, atol=1e-5) if precision == "fp32" else dict(rtol=2e-2, atol=2e-2)  # (x2 is exact in bf16 too)
        assert_close(g3, 2.0 * g1, what="scaled head", **tol)
        # perturb EVERY parameter (all packed copies must refresh: convs, fused skips, embedding banks, heads), then restore
        for p in m.parameters():
            p.mul_(1.25)
        e5, g5 = m(i["x"], t, i["z"])
        assert rel_l2(e5, e1) > 1e-2 and rel_l2(g5, g1) > 1e-2, "stale packed weights: output did not change"
        m.load_state_dict(sd)
        e4, g4 = m(i["x"], t, i["z"])
        assert_close(g4, g1, what="restored weights (grad)", **rep)
        assert_close(e4, e1, what="restored weights (eps)", **rep)


def test_oracle_agrees_on_gpu_inputs_at_larger_shape():
    """A shape with no recorded fixture: celeba64-proxy ShiftUNet, batch 2, vs the CPU oracle directly."""
    from pdae_b200.model.shift_unet import ShiftUNet
    from pdae_b200.utils.synth import fill_module_, synth_normal
    from tests.configs import CELEBA64_PROXY
    cfg = dict(CELEBA64_PROXY, latent_dim=512)
    m = fill_module_(ShiftUNet(**cfg), seed=21).eval()
    x, z = synth_normal((2, 3, 64, 64), 41), synth_normal((2, 512), 42)
    t = torch.tensor([17, 850])
    torch.set_num_threads(max(1, torch.get_num_threads()))
    with torch.no_grad():
        eps_ref, grad_ref = O.shiftunet_forward(cases.sd_of(m), cfg, x, t, z)
    m = m.cuda()
    for precision in ("fp32", "bf16", "bf16x3"):
        m.precision = precision
        with torch.no_grad():
            eps, grad = m(x.cuda(), t.cuda(), z.cuda())
        check(eps, eps_ref, precision, "celeba64-proxy eps")
        check(grad, grad_ref, precision, "celeba64-proxy grad")


@pytest.mark.parametrize("C,heads,new_order", [(128, 1, False), (128, 2, False), (128, 2, True), (256, 1, True)])
def test_attention_tensor_core(C, heads, new_order):
    """16x16 tokens (T=256): the bf16 path runs QK^T and PV as batched wgmma GEMMs -- vs the CPU oracle."""
    from pdae_b200.model import module as pm
    from pdae_b200.utils.synth import fill_module_, synth_normal
    m = fill_module_(pm.AttentionBlock(C, heads, -1, new_order), seed=31).eval()
    x = synth_normal((3, C, 16, 16), 32)
    sd = {"blk." + k: v for k, v in cases.sd_of(m).items()}
    ref = O.attention_block(sd, "blk", x, heads, new_order)
    m = m.cuda()
    for precision in ("fp32", "bf16", "bf16x3"):
        m.precision = precision
        with torch.no_grad():
            y = m(x.cuda())
        check(y, ref, precision, f"attention C={C} heads={heads} new={new_order}")
    plan3 = [v for k, v in m._plans().items() if k[1] == "bf16x3"][0][0]
    # split-operand mode: QK^T and PV as batched wgmma GEMMs on [hi|lo|hi] x [hi|hi|lo] operand blocks (fp32-grade)
    assert any(op[0] == "qkv_split3" for op in plan3.ops) and not any(op[0] == "attention_simt" for op in plan3.ops)
    plan = [v for k, v in m._plans().items() if k[1] == "bf16"][0][0]
    assert any(op[0].startswith("gemm_tc2") for op in plan.ops), "tensor-core attention path not taken"


@pytest.mark.parametrize("size,batch", [(24, 3), (48, 1), (40, 2)])
def test_ragged_resolutions_and_batches(size, batch):
    """Resolutions that are not powers of two (24 -> 12 -> 6, 48 -> 24 -> 12, 40 -> 20 -> 10: small or single-row tensor-core
    tiles, several images per tile with a masked batch tail, CUDA-core fallbacks) and odd batches, every precision mode."""
    from pdae_b200.model.shift_unet import ShiftUNet
    from pdae_b200.utils.synth import fill_module_, synth_normal
    cfg = dict(input_channel=3, base_channel=64, channel_multiplier=[1, 2, 2], num_residual_blocks_of_a_block=1,
               attention_resolutions=[2], num_heads=2, head_channel=-1, use_new_attention_order=False, dropout=0.0, latent_dim=128)
    m = fill_module_(ShiftUNet(**cfg), seed=41).eval()
    x, z = synth_normal((batch, 3, size, size), 42), synth_normal((batch, 128), 43)
    t = torch.tensor([5, 500, 999][:batch], dtype=torch.long)
    eps_ref, grad_ref = O.shiftunet_forward(cases.sd_of(m), cfg, x, t, z)
    m = m.cuda()
    for precision in ("fp32", "bf16x3", "bf16"):
        m.precision = precision
        with torch.no_grad():
            eps, grad = m(x.cuda(), t.cuda(), z.cuda())
        check(eps, eps_ref, precision, f"{size}x{size} B={batch} eps")
        check(grad, grad_ref, precision, f"{size}x{size} B={batch} grad")
