"""Times the two proposal operators that share the NMS kernels, and prints the card's name and power limit next to the
numbers, then one JSON line.

  mpt  ops.multi_proposal_target on the training step's shape: 16 chips of 32 x 32 x 21 anchors, NHWC, seeded RPN
       outputs (synth.mpt_inputs).
  mp   ops.multi_proposal on the Tester's largest ResNet-101 canvas (2 images, 84 x 128 x 21 anchors, 12000 pre-NMS
       rows) and on the MobileNetV2 one (2 images, 42 x 64 x 15, 6000), graph layout, tie-free and quantised scores
       (tests/multi_proposal_cases.py).
Each shape on both NMS paths (SNIPER_NMS_FAST=1 / 0): CUDA events around --launches calls after --warmup calls; the
median and the min of --repeats such windows, in microseconds per call.  --lib times another build of the library.

    python tools/multi_proposal_time.py [--launches 50] [--repeats 5] [--lib path/to/libsniper_b200.so]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from sniper_b200 import _lib, ops, synth  # noqa: E402


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip().replace("\n", " | ")


def window(fn, launches, warmup, repeats):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1000.0 / launches)
    return dict(median_us=float(np.median(out)), min_us=float(np.min(out)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--lib", default=None)
    a = ap.parse_args()
    if a.lib:
        _lib.LIB_PATH = os.path.abspath(a.lib)
    import multi_proposal_cases as C
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    shapes = {}
    cp, bp, im, gt, vr = synth.mpt_inputs(5, 16)
    mpt_in = [t(cp.transpose(0, 2, 3, 1)), t(bp.transpose(0, 2, 3, 1)), t(im), t(gt), t(vr)]
    shapes["mpt_b16_32x32"] = lambda: ops.multi_proposal_target(*mpt_in, layout=ops.NHWC)
    for name in ("resnet101-largest-tie_free", "resnet101-largest-quantised", "mobilenetv2-largest-tie_free",
                 "mobilenetv2-largest-quantised"):
        c = C.build(name)
        prob, head = C.device_inputs(c["cls_prob"], c["bbox_pred"], "graph", c["head_c"])
        args = (t(prob), t(head), t(c["im_info"]))
        shapes["mp_" + name] = (lambda args=args, c=c: ops.multi_proposal(*args, rpn_pre_nms_top_n=c["pre"],
                                                                          layout=ops.NHWC, **c["kw"]))
    res = dict(card=card(), lib=_lib.LIB_PATH)
    for fast in ("1", "0"):
        os.environ["SNIPER_NMS_FAST"] = fast
        for k, fn in shapes.items():
            r = window(fn, a.launches, a.warmup, a.repeats)
            res["%s_fast%s" % (k, fast)] = r
            print("%-40s SNIPER_NMS_FAST=%s  median %9.1f us  min %9.1f us" % (k, fast, r["median_us"], r["min_us"]))
    print(res["card"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
