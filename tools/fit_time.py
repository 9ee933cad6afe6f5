"""Times the training-metric kernel and Trainer.fit on one GPU; prints one JSON line.

  * sniper_train_metric_accum per launch at the ResNet-101 B = 20 and MobileNetV2 B = 40 step shapes (CUDA events over
    many queued launches) and its bytes/s against the bytes the step's tensors hold;
  * chips/s of fit (metrics on, Speedometer(20, 20)) against a per-step-synchronising step_raw loop over the same
    seeded roidb, alternated, `--runs` times each.

usage: python tools/fit_time.py [--runs 3] [--images 24] [--batch 20]
"""
import argparse
import json
import logging
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from sniper_b200 import callback, metric, model, ops, trainer  # noqa: E402
from sniper_b200 import iterator as IT  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def kernel_time(B, H, A, N, K, iters=2000):
    dev = "cuda:0"
    g = torch.Generator(device=dev).manual_seed(0)
    prob = torch.rand(B, H, H, 2 * A, device=dev, generator=g)
    label = torch.randint(-1, 2, (B, A * H * H), device=dev, generator=g).float()
    cls = torch.rand(N, K, device=dev, generator=g)
    clab = torch.randint(-1, K, (N,), device=dev, generator=g).float()
    counts = torch.tensor([int((label != -1).sum()), int((clab != -1).sum())], dtype=torch.int32, device=dev)
    loss = torch.zeros(8, device=dev)
    acc = metric.MetricAccumulator(dev)
    for _ in range(50):
        ops.train_metric_accum(prob, label, A, cls, clab, counts, loss, acc.buf, acc.workspace)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.train_metric_accum(prob, label, A, cls, clab, counts, loss, acc.buf, acc.workspace)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    nbytes = 4 * (prob.numel() + label.numel() + cls.numel() + clab.numel())
    return dict(us_per_launch=round(us, 2), mbytes=round(nbytes / 1e6, 2), gbytes_per_s=round(nbytes / us / 1e3, 1))


def fit_run(tr, roidb, cfg, B, use_fit):
    np.random.seed(1)
    it = IT.MNIteratorE2E([dict(r) for r in roidb], cfg, batch_size=B, n_buffers=6)
    stage = IT.InputStage(cfg, "cuda:0", B)
    pf = IT.PrefetchingIter(it, depth=2, epochs=1, epoch_marker=use_fit)
    n = 0
    try:
        torch.cuda.synchronize()
        t0 = time.time()
        if use_fit:
            tr.fit(pf, stage, 1, batch_end_callback=callback.Speedometer(B, 20))
            n = None
        else:
            for raw in pf:
                tr.step_raw(raw, stage)
                n += 1
        torch.cuda.synchronize()
        dt = time.time() - t0
    finally:
        pf.close()
    return dt, it.size if n is None else n * B


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--images", type=int, default=24)
    ap.add_argument("--batch", type=int, default=20)
    a = ap.parse_args()
    logging.basicConfig(level=logging.INFO, stream=sys.stderr)
    res = {"card": card(), "kernel": {"resnet101_b20": kernel_time(20, 32, 21, 6000, 81),
                                      "mobilenetv2_b40": kernel_time(40, 16, 15, 12000, 81)}}
    cfg = IT.default_config()
    roidb = IT.synthetic_roidb(a.images, seed=3)
    mc = model.Cfg()
    mc.batch_images = a.batch
    # both loops run the same captured graphs, metric launch included: they differ in the per-step synchronisation
    tr = trainer.Trainer(mc, device="cuda:0", scheduler=None, metrics=True)
    fit_run(tr, roidb, cfg, a.batch, False)          # warm-up: capture, module loading
    rates = {"fit": [], "step_raw": []}
    for _ in range(a.runs):
        for name in ("step_raw", "fit"):
            dt, chips = fit_run(tr, roidb, cfg, a.batch, name == "fit")
            rates[name].append(round(chips / dt, 2))
    res["chips_per_s"] = rates
    res["images"], res["batch"] = a.images, a.batch
    print(json.dumps(res))


if __name__ == "__main__":
    main()
