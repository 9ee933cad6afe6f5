"""Times the HBM-bound BatchNorm kernels alone (CUDA-graph replay of 20 launches over rotating buffers larger than L2)
and prints algorithmic GB/s.  Usage: [GT_DTYPE=bf16] python tools/ew_time.py"""
import os
import sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sniper_b200 import ops

DT = torch.bfloat16 if os.environ.get("GT_DTYPE") == "bf16" else torch.float32
ES = 2 if DT == torch.bfloat16 else 4
SHAPES = [(20480, 256), (20480, 1024), (81920, 128), (81920, 512), (327680, 64), (327680, 256)]


def timed(fn, reps=20):
    for i in range(3):
        fn(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        with torch.cuda.graph(g, stream=st):
            for i in range(reps):
                fn(i)
    ts = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); g.replay(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[2] * 1e3 / reps


for M, C in SHAPES:
    nbuf = max(3, int(400e6 // (M * C * ES)) + 1)
    X = [torch.randn(M, C, device="cuda").to(DT) for _ in range(nbuf)]
    DY = [torch.randn(M, C, device="cuda").to(DT) for _ in range(nbuf)]
    Y = [torch.empty(M, C, device="cuda", dtype=DT) for _ in range(nbuf)]
    bn = ops.BNState(C, "cuda")
    bn.dgamma = torch.zeros(C, device="cuda"); bn.dbeta = torch.zeros(C, device="cuda")
    ops.bn_stats(X[0], bn)
    byts = M * C * ES
    cases = {
        "stats(1r)": (lambda i: ops.bn_stats(X[i % nbuf], bn), 1),
        "apply(1r1w)": (lambda i: ops.affine_act(X[i % nbuf], bn.scale, bn.shift, relu=True, out=Y[i % nbuf]), 2),
        "bwd(4r1w)": (lambda i: ops.bn_relu_bwd(X[i % nbuf], DY[i % nbuf], bn, out=Y[i % nbuf]), 5),
        "bwd+add(5r1w)": (lambda i: ops.bn_relu_bwd(X[i % nbuf], DY[i % nbuf], bn, add=DY[(i + 1) % nbuf], out=Y[i % nbuf]), 6),
    }
    for name, (fn, passes) in cases.items():
        us = timed(fn)
        print("%7d x %4d %-14s %.1f us %.2f TB/s" % (M, C, name, us, passes * byts / us / 1e6), flush=True)
    del X, DY, Y
