"""Cost of the deterministic plans' batch-invariant partitioning, at B = 1, 8 and 256 (switch on throughout):
  * ch_stats_det and gn_stats_det (ch_parts + the ordered slot reduction) on the celeba64-proxy levels, CUDA events over
    --reps launches each;
  * one deterministic decoder step (the ShiftUNet plan_for plan replayed as one CUDA graph), celeba64-proxy, "bf16x3" and
    "bf16".
--root DIR times another checkout's package (e.g. the parent commit), so two versions can alternate on one card.
usage: python scripts/batch_invariance_bench.py [--root DIR] [--reps N] [--out FILE]   (card name and power limit in the output)"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def events_ms(fn, reps):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def stats_rows(reps):
    import torch
    from pdae_b200 import _native
    L = _native.lib()
    dev = torch.device("cuda")
    rows = []
    for S, C in ((64, 64), (32, 128), (16, 256), (8, 512), (4, 512)):
        for B in (1, 8, 256):
            HW = S * S
            x = torch.randn(B, HW, C, device=dev)
            ws = torch.empty(int(L.pdae_stats_det_workspace_bytes(B, HW, C)) // 4 + 4, device=dev)
            chs = torch.empty(B, C, 2, device=dev)
            sums = torch.empty(B, 32, 2, device=dev, dtype=torch.float64)
            st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

            def ch():
                _native.check(L.pdae_ch_stats_det(x.data_ptr(), B, HW, C, chs.data_ptr(), ws.data_ptr(), ws.numel() * 4, st),
                              "ch_stats_det")

            def gn():
                _native.check(L.pdae_gn_stats_det(x.data_ptr(), C, None, 0, B, HW, sums.data_ptr(), ws.data_ptr(), ws.numel() * 4,
                                                  st), "gn_stats_det")
            rows.append({"op": "ch_stats_det", "level": f"{S}x{S}", "C": C, "B": B, "us": round(1e3 * events_ms(ch, reps), 2)})
            rows.append({"op": "gn_stats_det", "level": f"{S}x{S}", "C": C, "B": B, "us": round(1e3 * events_ms(gn, reps), 2)})
    return rows


def step_rows(reps):
    import torch
    from bench import WORKLOADS
    from pdae_b200.model.shift_unet import ShiftUNet
    from pdae_b200.utils.synth import fill_module_, synth_normal
    dev = torch.device("cuda")
    cfg, size = WORKLOADS["celeba64"][0], WORKLOADS["celeba64"][1]
    rows = []
    for precision in ("bf16x3", "bf16"):
        dec = fill_module_(ShiftUNet(latent_dim=512, **cfg), seed=0).eval().to(dev)
        dec.precision = precision
        for B in (1, 8, 256):
            x, z = synth_normal((B, 3, size, size), 1).to(dev), synth_normal((B, 512), 2).to(dev)
            t = torch.full((B,), 500, device=dev, dtype=torch.long)
            with torch.no_grad():
                dec(x, t, z)
            plan, _ = dec.plan_for(B, size, size)
            assert plan.det
            plan.capture_graph()
            ms = events_ms(lambda: plan.run(prologue=False), reps if B < 256 else max(3, reps // 4))
            rows.append({"op": f"decoder step celeba64-proxy {precision}", "B": B, "ms": round(ms, 4)})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=HERE, help="checkout whose pdae_b200 package is timed")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sys.path.insert(0, HERE)                     # bench.WORKLOADS
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    torch.use_deterministic_algorithms(True, warn_only=True)
    gpu = card()
    rows = stats_rows(args.reps) + step_rows(max(5, args.reps // 10))
    for r in rows:
        r.update(root=os.path.abspath(args.root), card=gpu)
        print(json.dumps(r), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
