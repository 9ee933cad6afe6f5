"""Algorithmic bytes and lower bounds of the wgmma launches of one training step, from `bench.py`'s per-shape table.

    SNIPER_DUMP_GEMM=gemm.md python bench.py --gpus 1 --steps 10 --warmup 3
    python tools/gemm_shapes.py gemm.md [gemm_other.md]

For every row of the table (kind, M, N, K, operand type, launches, total ms) this adds the bytes the launch must move
through HBM at least, its arithmetic intensity and the lower bound max(FLOP / tensor peak, bytes / HBM bandwidth) at the
H100 SXM data-sheet rates (495 TFLOP/s TF32, 989 bf16, 3.35 TB/s), then sums the launches per class:

  * K-major (gemm, conv) whose intensity is under the ridge point peak / bandwidth: HBM-bound;
  * K-major at or over the ridge point: tensor-bound;
  * weight gradients (wgrad, MN-major operands).

Bytes per launch (fp32 storage for tf32 operands, 2 bytes for bf16): the A operand once (a convolution reads its input
once, M x K / taps elements, with taps = 9 when K is 9 x a multiple of 32 channels, else 1), B once, the output once
(weight gradients read and write their fp32 dW).  A residual or an accumulated output adds to that; the table does not
say which launches have one, so the bound stays a lower bound.

With a second table (the same step on another build) the rows are matched by shape and shown side by side.
"""
import re
import sys

PEAK_TFLOPS = {"tf32": 495.0, "bf16": 989.0}
HBM_TBS = 3.35


def read_table(path):
    rows = {}
    for line in open(path):
        m = re.match(r"\|\s*(gemm|conv|wgrad)\s*\|\s*(\d+)\s*\|\s*(\d+)\s*\|\s*(\d+)\s*\|\s*(tf32|bf16)\s*\|\s*(\d+)\s*\|"
                     r"\s*([\d.]+)\s*\|", line)
        if m:
            kind, M, N, K, dt, n, ms = m.groups()
            rows[(kind, int(M), int(N), int(K), dt)] = (int(n), float(ms))
    return rows


def launch_bytes(kind, M, N, K, dt):
    esz = 4 if dt == "tf32" else 2
    if kind == "wgrad":
        # M = Cout, N = taps * Cin, K = pixels
        taps = 9 if N % 9 == 0 and (N // 9) % 32 == 0 else 1
        return esz * (K * M + K * N // taps) + 8 * M * N
    taps = 9 if kind == "conv" and K % 9 == 0 and (K // 9) % 32 == 0 else 1
    return esz * (M * K // taps + N * K + M * N)


def describe(key):
    kind, M, N, K, dt = key
    flops = 2.0 * M * N * K
    nbytes = launch_bytes(*key)
    ridge = PEAK_TFLOPS[dt] / HBM_TBS
    intensity = flops / nbytes
    t_tc = flops / (PEAK_TFLOPS[dt] * 1e12) * 1e3
    t_hbm = nbytes / (HBM_TBS * 1e12) * 1e3
    if kind == "wgrad":
        cls = "weight gradient"
    else:
        cls = "K-major, HBM-bound" if intensity < ridge else "K-major, tensor-bound"
    return dict(flops=flops, bytes=nbytes, intensity=intensity, bound_ms=max(t_tc, t_hbm), cls=cls)


def main(paths):
    tables = [read_table(p) for p in paths]
    keys = sorted(set().union(*tables), key=lambda k: -tables[0].get(k, (0, 0.0))[1])
    head = "| class | kind | M | N | K | operands | launches | MB / launch | FLOP/B | bound ms |"
    for i in range(len(tables)):
        head += " ms [%d] | TFLOP/s [%d] | GB/s [%d] |" % (i, i, i)
    print(head)
    print("|" + "---|" * (head.count("|") - 1))
    classes = {}
    for k in keys:
        d = describe(k)
        n = max(t.get(k, (0, 0.0))[0] for t in tables)
        line = "| %s | %s | %d | %d | %d | %s | %d | %.1f | %.0f | %.3f |" % (
            d["cls"], k[0], k[1], k[2], k[3], k[4], n, d["bytes"] / 1e6, d["intensity"], n * d["bound_ms"])
        c = classes.setdefault(d["cls"], [0, 0.0, 0.0, 0.0, [0.0] * len(tables)])
        c[0] += n; c[1] += n * d["flops"]; c[2] += n * d["bytes"]; c[3] += n * d["bound_ms"]
        for i, t in enumerate(tables):
            if k in t:
                ln, ms = t[k]
                c[4][i] += ms
                line += " %.3f | %.1f | %.0f |" % (ms, ln * d["flops"] / (ms / 1e3) / 1e12, ln * d["bytes"] / (ms / 1e3) / 1e9)
            else:
                line += " - | - | - |"
        print(line)
    print()
    print("| class | launches | GFLOP | GB | lower bound ms |" + "".join(" ms [%d] |" % i for i in range(len(tables))))
    print("|---|---:|---:|---:|---:|" + "---:|" * len(tables))
    for cls, (n, fl, nb, b, ms) in sorted(classes.items()):
        print("| %s | %d | %.0f | %.1f | %.1f |" % (cls, n, fl / 1e9, nb / 1e9, b) + "".join(" %.1f |" % m for m in ms))


if __name__ == "__main__":
    if len(sys.argv) < 2:
        raise SystemExit(__doc__)
    main(sys.argv[1:])
