"""Time conv_tc3 (fused-prologue conv) in isolation through the C-ABI, rotating over several buffer sets (L2-cold-ish).
usage: python scripts/conv3_bench.py B H W C1 C2 Cout x3(0/1) res(0/1) skip(0/1) [bn]"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from pdae_b200 import _native
from pdae_b200._native import PDAE_BF16, PDAE_F32

B, H, W, C1, C2, Cout, x3, res, skip = (int(a) for a in sys.argv[1:10])
bn = int(sys.argv[10]) if len(sys.argv) > 10 else 0
dev = "cuda"
L = _native.lib()
P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
Cin = C1 + C2
sdt = torch.float32 if x3 else torch.bfloat16
odt = torch.float32 if x3 else torch.bfloat16
nmat = 2 if x3 else 1
w = torch.randn(9, nmat, Cout, Cin, device=dev).to(torch.bfloat16).contiguous()
wsk = torch.randn(nmat, Cout, Cin, device=dev).to(torch.bfloat16).contiguous() if skip else None
bias = torch.randn(Cout, device=dev)
nset = 4
plans, keep = [], []
for i in range(nset):
    s1 = torch.randn(B, H, W, C1, device=dev).to(sdt)
    s2 = torch.randn(B, H, W, C2, device=dev).to(sdt) if C2 else None
    ab = torch.randn(B, 2, Cin, device=dev)
    r = torch.randn(B, H, W, Cout, device=dev).to(odt) if res else None
    out = torch.empty(B, H, W, Cout, device=dev, dtype=odt)
    st = torch.zeros(B, Cout, 2, device=dev)
    h = ctypes.c_void_p()
    rc = L.pdae_conv_tc3_create(ctypes.byref(h), P(s1), C1, P(s2), C2, PDAE_F32 if x3 else PDAE_BF16, P(ab), 1, P(w), P(bias),
                                P(s1) if skip else None, C1 if skip else 0, P(s2) if skip and C2 else None, C2 if skip else 0,
                                P(wsk), P(r), P(out), PDAE_F32 if x3 else PDAE_BF16, P(st), B, H, W, Cout, bn)
    _native.check(rc, "create")
    plans.append(h)
    keep.append((s1, s2, ab, r, out, st))
stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
for h in plans:
    _native.check(L.pdae_conv_tc3_run(h, stream), "run")
torch.cuda.synchronize()
reps = 5
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(reps):
    for h in plans:
        L.pdae_conv_tc3_run(h, stream)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / (reps * nset)
fl = 2.0 * B * H * W * Cout * (Cin * 9 + (Cin if skip else 0))
print(f"conv_tc3 {B}x{H}x{W} {C1}+{C2}->{Cout} x3={x3} res={res} skip={skip} bn={bn}: "
      f"{ms * 1e3:.1f} us  {fl / ms / 1e9:.1f} TFLOP/s (algorithmic)")
