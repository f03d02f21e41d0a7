"""Time one tensor-core conv in isolation (L2-cold between reps by rotating over several buffer sets).
usage: python scripts/conv_bench.py B H W Cin Cout k res(0/1) out_bf16(0/1) stats(0/1) [bn]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from pdae_b200.engine import Plan

B, H, W, Cin, Cout, k, res, obf, stats = (int(a) for a in sys.argv[1:10])
bn = int(sys.argv[10]) if len(sys.argv) > 10 else 0
dev = torch.device("cuda")
nset = 4
plans = []
w = (torch.randn(Cout, Cin, k, k, device=dev) / (Cin * k * k) ** 0.5)
bias = torch.randn(Cout, device=dev)
for i in range(nset):
    P = Plan(dev, "bf16")
    x = torch.randn(B, H, W, Cin, device=dev).to(torch.bfloat16)
    out = P.new((B, H, W, Cout), torch.bfloat16 if obf else torch.float32)
    out.keep = True
    r = P.fixed(torch.randn(B, H, W, Cout, device=dev)) if res else None
    P.conv(P.fixed(x), w, bias, out, B=B, H=H, W=W, Cin=Cin, Cout=Cout, k=k, residual=r, want_stats=bool(stats), bn_override=bn)
    P.finalize()
    plans.append(P)
for P in plans:
    P.run()
torch.cuda.synchronize()
reps = 5
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(reps):
    for P in plans:
        P.run()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / (reps * nset)
fl = 2.0 * B * H * W * Cout * Cin * k * k
byts = B * H * W * (Cin * 2 + Cout * (2 if obf else 4) + (Cout * 4 if res else 0))
print(f"conv {B}x{H}x{W} {Cin}->{Cout} k{k} res={res} obf16={obf} stats={stats} bn={bn}: {ms * 1e3:.1f} us  "
      f"{fl / ms / 1e9:.1f} TFLOP/s  {byts / ms / 1e6:.0f} GB/s (algorithmic bytes)")
