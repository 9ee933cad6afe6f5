"""Builds sniper_b200/lib/libsniper_b200.so (sm_90a) in-tree with nvcc.  No torch involved."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libsniper_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-ffp-contract=off", "-Xcompiler", "-fopenmp",
    "--expt-relaxed-constexpr", "-split-compile", "0",
]
# translation units whose results are graded bit-exact: no FMA contraction anywhere
NO_FMAD = {"mpt.cu", "psroi.cu", "anchor_target.cu", "nms.cu", "coco_eval.cu", "detect_post.cu", "train_metric.cu",
           "voc_eval.cu", "proposal_recall.cu", "focus_chips.cu", "chip_plan.cu"}


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))


def build(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    objs = []
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(HERE, "..", "include", "sniper_b200.h"))
    newest_hdr = max([os.path.getmtime(h) for h in hdrs if os.path.exists(h)] + [0])
    procs = []
    for f in sources():
        src = os.path.join(CSRC, f)
        obj = os.path.join(LIBDIR, f + ".o")
        objs.append(obj)
        if (not force and os.path.exists(obj) and os.path.getmtime(obj) > os.path.getmtime(src)
                and os.path.getmtime(obj) > newest_hdr):
            continue
        cmd = ["nvcc"] + NVCC_FLAGS + (["-fmad=false"] if f in NO_FMAD else []) + (
            ["-Xptxas", "-v"] if verbose else []) + ["-x", "cu", "-I", os.path.join(HERE, "..", "include"),
                                                     "-c", src, "-o", obj]
        procs.append((f, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for f, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0 or verbose:
            sys.stderr.write("== %s\n%s\n" % (f, out))
        failed |= pr.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    if procs or not os.path.exists(LIB):
        cmd = ["nvcc", "-shared", "-o", LIB] + objs + ["-Xcompiler", "-fopenmp", "-lgomp"]
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
