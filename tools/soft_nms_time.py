"""Times the batched device soft-NMS (sniper_soft_nms_batched) on runs shaped like BASELINE config 5's aggregation --
80 classes x a few images in one launch, most problems small or empty, a few of up to a few thousand rows -- and prints
the card's name and power limit next to the numbers, then one JSON line.

  saturated  rows of a saturated softmax (10-30 % of the scores at exactly 1.0f) with duplicated rows, as three scales
             of overlapping chips give them (tests/soft_nms_cases.py)
  tie_free   the same boxes with distinct scores
  heavy      tight clusters of low scores: most rows leave in the first rounds
  sparse     saturated rows, but at most 19 per problem and most problems empty (a run whose detector fires rarely,
             such as bench.py --config5 with its random-init weights: some 200 detections per image)
Gaussian (sigma 0.55, Nt 0.3, threshold 0.001, as inference.aggregate calls it).  Every --lib is loaded into the same
process and the libraries are timed alternately: CUDA events around --launches calls after --warmup calls, --repeats
windows per library; median and min in microseconds per launch, each including the copy of the input rows into the
output buffer the kernel rewrites in place (as ops.soft_nms_batched clones them).  Also counts the problems whose output differs from
the first library's.

    python tools/soft_nms_time.py [--lib A.so --lib B.so] [--images 4] [--launches 20] [--repeats 7]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from sniper_b200 import _lib  # noqa: E402


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip().replace("\n", " | ")


def load(path):
    """sniper_soft_nms_batched of the library at `path`, loaded on its own (not through _lib's singleton)."""
    fn = ctypes.CDLL(os.path.abspath(path)).sniper_soft_nms_batched
    res, args = _lib.SIGNATURES["sniper_soft_nms_batched"]
    fn.restype, fn.argtypes = _lib._T[res], [_lib._T[c] for c in args]
    return fn


def run_set(kind, images, seed):
    """[total,5] rows and int32 offsets of 80 classes x `images` problems (class-major within an image)."""
    import soft_nms_cases as C
    rng = np.random.RandomState(seed)
    probs = []
    for _ in range(images * 80):
        u = rng.rand()
        if kind == "sparse":
            n = 0 if u < 0.6 else int(rng.randint(1, 20))
        else:
            n = 0 if u < 0.4 else int(rng.randint(1, 40)) if u < 0.85 else int(np.exp(rng.uniform(np.log(40),
                                                                                                  np.log(3000))))
        if n == 0:
            probs.append(np.zeros((0, 5), np.float32))
        elif kind == "heavy":
            probs.append(C._rows("heavy_decay", rng, n))
        else:
            d = C._aggregated(rng, n).copy()
            if kind == "tie_free":
                d[:, 4] = C._tie_free(rng, n)
            probs.append(d)
    sizes = [len(d) for d in probs]
    return np.concatenate(probs, 0), np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="library to time (repeatable; default: the built one)")
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=7)
    a = ap.parse_args()
    libs = a.lib or [_lib.LIB_PATH]
    fns = [load(p) for p in libs]
    res = dict(card=card(), libs=libs, images=a.images, sets={})
    stream = torch.cuda.current_stream()
    for k, kind in enumerate(("saturated", "tie_free", "heavy", "sparse")):
        rows, offsets = run_set(kind, a.images, 100 + k)
        P = len(offsets) - 1
        dets = torch.from_numpy(rows).cuda()
        off = torch.from_numpy(offsets).cuda()
        outs = [dets.clone() for _ in fns]
        counts = [torch.zeros(P, dtype=torch.int32, device="cuda") for _ in fns]
        scratch = torch.empty((rows.shape[0], 6), dtype=torch.float32, device="cuda")

        def call(li):
            outs[li].copy_(dets)
            _lib.check(fns[li](outs[li].data_ptr(), off.data_ptr(), P, 0.55, 0.3, 0.001, 2, counts[li].data_ptr(),
                               scratch.data_ptr(), stream.cuda_stream))
        for li in range(len(fns)):
            for _ in range(a.warmup):
                call(li)
        torch.cuda.synchronize()
        times = [[] for _ in fns]
        for _ in range(a.repeats):
            for li in range(len(fns)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.launches):
                    call(li)
                e1.record()
                torch.cuda.synchronize()
                times[li].append(e0.elapsed_time(e1) * 1000.0 / a.launches)
        c0, o0 = counts[0].cpu().numpy(), outs[0].cpu().numpy()
        entry = dict(problems=P, rows=int(rows.shape[0]), largest=int(np.diff(offsets).max()), libs=[])
        for li, p in enumerate(libs):
            c, o = counts[li].cpu().numpy(), outs[li].cpu().numpy()
            differ = sum(1 for q in range(P) if c[q] != c0[q] or not np.array_equal(
                o[offsets[q]:offsets[q] + c[q]], o0[offsets[q]:offsets[q] + c0[q]]))
            r = dict(lib=p, median_us=float(np.median(times[li])), min_us=float(np.min(times[li])),
                     problems_differing_from_first=differ)
            entry["libs"].append(r)
            print("%-10s %6d rows (largest %4d)  %-50s median %9.1f us  min %9.1f us  %d problems differ" % (
                kind, entry["rows"], entry["largest"], p[-50:], r["median_us"], r["min_us"], differ))
        res["sets"][kind] = entry
    print(res["card"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
