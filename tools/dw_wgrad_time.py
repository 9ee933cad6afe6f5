"""Per-shape time of the depthwise 3x3 weight gradient at every inverted-residual unit of the MobileNetV2 training step
(BASELINE config 4), and its total per step.

    python tools/dw_wgrad_time.py [--B 40] [--fp32] [--reps 50] [--root TREE]

Each shape is timed with CUDA events over `reps` back-to-back calls of ops.depthwise3x3_wgrad (inputs resident, after
warm-up) and reported with the algorithmic traffic (x + dy read once).  --root imports the package from another
checkout, so two builds can be compared in one process run each.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys


def unit_shapes(MM, B, chip=512):
    cfg = MM.MCfg()
    H = (chip - 1) // 2 + 1
    out, cin = [], cfg.first_c
    for t, c, n, s in cfg.bottlenecks:
        for j in range(n):
            e = int(round((cin if j == 0 else c) * t))
            st = s if j == 0 else 1
            out.append((B, H, H, MM.pad64(e), st))
            H = (H - 1) // st + 1
        cin = c
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=40)
    ap.add_argument("--fp32", action="store_true")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from sniper_b200 import model_mnv2 as MM
    from sniper_b200 import ops
    assert torch.cuda.is_available(), "needs a CUDA device"
    dt = torch.float32 if args.fp32 else torch.bfloat16
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    rows, total = [], 0.0
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    for NB, H, W, C, s in unit_shapes(MM, args.B):
        Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
        x = torch.randn(NB, H, W, C, device="cuda", generator=g).to(dt)
        dy = torch.randn(NB, Ho, Wo, C, device="cuda", generator=g).to(dt)
        dw = torch.zeros(9, C, device="cuda")
        for _ in range(5):
            ops.depthwise3x3_wgrad(x, dy, dw, s)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            ops.depthwise3x3_wgrad(x, dy, dw, s)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / args.reps
        nbytes = (x.numel() + dy.numel()) * x.element_size()
        rows.append({"shape": "%dx%dx%dx%d s%d" % (NB, H, W, C, s), "us": round(us, 1), "gbs": round(nbytes / us / 1e3, 1)})
        total += us
        del x, dy
    print(json.dumps({"root": os.path.abspath(args.root), "dtype": "fp32" if args.fp32 else "bf16", "B": args.B,
                      "gpu": gpu, "total_us_per_step": round(total, 1), "shapes": rows}))


if __name__ == "__main__":
    main()
