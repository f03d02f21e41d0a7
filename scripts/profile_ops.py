"""Per-op device times of one ShiftUNet decoder step (CUDA events around every launch; warm L2, no graph).
usage: python scripts/profile_ops.py [workload] [batch] [top_n] [precision]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import pdae_b200
from bench import WORKLOADS
from pdae_b200.model.shift_unet import ShiftUNet
from pdae_b200.utils.synth import fill_module_, synth_normal

wl = sys.argv[1] if len(sys.argv) > 1 else "celeba64"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 256
top = int(sys.argv[3]) if len(sys.argv) > 3 else 40
prec = sys.argv[4] if len(sys.argv) > 4 else "bf16"
cfg, size = WORKLOADS[wl][0], WORKLOADS[wl][1]
pdae_b200.set_default_precision(prec)
dev = torch.device("cuda")
dec = fill_module_(ShiftUNet(latent_dim=512, **cfg), seed=0).eval().to(dev)
x = synth_normal((B, 3, size, size), 1).to(dev)
z = synth_normal((B, 512), 2).to(dev)
t = torch.full((B,), 500, device=dev, dtype=torch.long)
with torch.no_grad():
    dec(x, t, z)
plan, _ = dec.plan_for(B, size, size)
prof = plan.profile(reps=5)
tot = sum(v["ms"] for v in prof.values())
print(f"workload {wl} B={B} {prec}: sum of op times {tot:.2f} ms, {len(plan.ops)} ops")
for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"]):
    tf = v["flops"] / (v["ms"] * 1e9) if v["flops"] else 0
    print(f"  {k:18s} {v['ms']:8.3f} ms  {100 * v['ms'] / tot:5.1f}%  n={v['launches']:4d}  {tf:8.1f} TFLOP/s")
rows = []
for i, (fn, args) in enumerate(plan.ops):
    if fn == "conv_tc3":
        (s1, C1, s2, C2, sdt, ab, silu, w, bias, k1, S1, k2, S2, wsk, resid, out, odt, stats, Bb, H, W, Cout, bn) = args
        rows.append((plan.last_op_ms[i], f"conv_tc3 {H}x{W} {C1}+{C2}->{Cout} skip={S1 + S2} res={int(resid is not None)} obf16={odt}",
                     plan.flops[i]))
    elif fn.startswith("conv_tc2"):
        ints = [a for a in args if isinstance(a, int)]
        if fn == "conv_tc2_skip":
            odt, Bb, H, W, Cin, Cout, k, bn = ints[-8:]
            cv = 0
            fn = f"conv_tc2+skip{ints[0]}"
        else:
            odt, Bb, H, W, Cin, Cout, k, cv, bn = ints[-9:]
        res = args[3] is not None
        rows.append((plan.last_op_ms[i], f"{fn} {H}x{W} {Cin}->{Cout} k{k} res={int(res)} obf16={odt} head={cv}", plan.flops[i]))
agg = {}
for ms, key, fl in rows:
    a = agg.setdefault(key, [0, 0.0, 0.0])
    a[0] += 1; a[1] += ms; a[2] += fl
print("conv shapes by total time:")
for key, (n, ms, fl) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:top]:
    print(f"  {key:58s} n={n:3d} {ms:8.3f} ms  avg {1e3 * ms / n:8.1f} us  {fl / (ms * 1e9):7.1f} TFLOP/s")

print("gn_apply by total time:")
agg = {}
for i, (fn, args) in enumerate(plan.ops):
    if fn == "gn_apply":
        src1, sdt, C1, src2, sdt2, C2, ab, silu, rs, Bb, H, W, act, adt, raw, rdt = args[:16]
        C = C1 + C2
        Ho, Wo = (2 * H, 2 * W) if rs == 1 else ((H // 2, W // 2) if rs == 2 else (H, W))
        rd = Bb * H * W * (C1 * (2 if sdt == 1 else 4) + C2 * (2 if sdt2 == 1 else 4))
        wr = Bb * Ho * Wo * C * ((2 if adt == 1 else 4) + (0 if raw is None else (2 if rdt == 1 else 4)))
        key = f"{H}x{W} C={C1}+{C2} src={'bf16' if sdt else 'f32'}/{'bf16' if sdt2 else 'f32'} rs={rs} raw={0 if raw is None else (2 if rdt == 1 else 4)}"
        a = agg.setdefault(key, [0, 0.0, 0])
        a[0] += 1; a[1] += plan.last_op_ms[i]; a[2] += rd + wr
for key, (n, ms, by) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:14]:
    print(f"  {key:48s} n={n:3d} {ms:7.3f} ms avg {1e3 * ms / n:7.1f} us  {by / ms / 1e6:7.0f} GB/s")
