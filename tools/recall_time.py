"""Times proposal recall (recall.evaluate_recall) on a seeded COCO-train-shaped set and prints one JSON line.

The set: --images images (default 20 000), 1000-3000 float32 proposals and about 7 uint16 GTs per image (some over 256^2
in area, 3% crowd rows), 1% of the images with 60-100 GTs.  Reported, with the card's name, power limit and max SM
clock read in the same run:
  kernel_ms      the matching and accumulation kernels (torch.profiler CUDA activity, summed, one warmed call)
  call_ms        ops.proposal_recall end to end (host CSR in, host results out; CUDA events, mean of --repeat)
  evaluate_s     recall.evaluate_recall end to end, roidb in, string out (host wall clock, mean of --repeat)
  numpy_s        the numpy restatement (oracle/recall_np.py) on --np-images images, and that time scaled to the set
Usage: python tools/recall_time.py [--images N] [--np-images N] [--repeat N]"""
import argparse
import json
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", "tests"))
sys.path.insert(0, os.path.join(HERE, "..", "oracle"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=20000)
    ap.add_argument("--np-images", type=int, default=500)
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("recall_time.py needs a CUDA device")
    import recall_fixture as F
    import recall_np
    from sniper_b200 import ops, recall
    roidb, cand = F.coco_like(2024, a.images)
    thr = recall.default_thresholds()
    inputs = recall.recall_inputs(roidb, cand)
    res = ops.proposal_recall(*inputs, thr)                        # warm-up
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ops.proposal_recall(*inputs, thr)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "recall_" in e.name:
            k = "match" if "match" in e.name else "accumulate"
            kern[k] = kern.get(k, 0.0) + e.device_time_total / 1e3
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(a.repeat):
        ops.proposal_recall(*inputs, thr)
    ev1.record()
    torch.cuda.synchronize()
    call_ms = ev0.elapsed_time(ev1) / a.repeat
    t0 = time.time()
    for _ in range(a.repeat):
        text = recall.evaluate_recall(roidb, cand, verbose=False)
    torch.cuda.synchronize()
    evaluate_s = (time.time() - t0) / a.repeat
    t0 = time.time()
    np_text, _ = recall_np.evaluate(roidb[:a.np_images], cand[:a.np_images])
    numpy_s = time.time() - t0
    dev_text = recall.evaluate_recall(roidb, cand, num_images=a.np_images, verbose=False)
    print(json.dumps(dict(
        card=card(), images=a.images, proposals=int(inputs[1][-1]), gts=int(inputs[3][-1]),
        kernel_ms=kern, call_ms=round(call_ms, 3),
        evaluate_s=round(evaluate_s, 3), numpy_images=a.np_images, numpy_s=round(numpy_s, 3),
        numpy_s_scaled=round(numpy_s * a.images / a.np_images, 1), subset_equal=np_text == dev_text,
        ar_all=float(res['ar'][0]), text_head=text[:60])))


if __name__ == "__main__":
    main()
