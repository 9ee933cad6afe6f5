"""Times the training epoch plan, `MNIteratorE2E.reset()`, with the host chip_worker and with the device plan
(`plan_backend="device"`) side by side, and prints the card's name, power limit and max SM clock next to the numbers,
then one JSON line.

  workload  seeded, COCO-train shaped synthetic roidbs (`iterator.synthetic_roidb` without pixels: 1333 x 800 or
            800 x 1333, 1-20 GTs): GT only (no negative chips), 300 and 1000 proposals per image with negative chips;
            the default resolution scales and the paper's factor scales (`load_data.PAPER_COCO_SCALES`); and one roidb
            with a flipped copy of every entry.
  reset     host and device `reset()` alternated, --repeats runs each, host clock around the whole call (the device plan
            synchronises its stream before it returns); both plans are compared first (plan digest).  Reported per
            image, with the device plan's CUDA-event time of its launches, its H2D bytes per epoch, the device bytes it
            keeps between epochs and the peak device memory of an epoch.
  replay    a resumed run (`--begin-epoch 3`): iterator construction plus three resets, host against device.

    python tools/plan_time.py [--images 400] [--repeats 2]
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from sniper_b200 import host, iterator as IT, load_data  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:                                 # noqa: BLE001
        q = torch.cuda.get_device_name(0)
    return q


def roidb(n, n_prop, flipped, seed=0):
    out = [{k: v for k, v in r.items() if k != 'image_data'}
           for r in IT.synthetic_roidb(n, seed=seed, n_prop=n_prop)]
    if flipped:
        for r in list(out):
            b = r['boxes'].copy()
            b[:, 0], b[:, 2] = r['width'] - r['boxes'][:, 2] - 1, r['width'] - r['boxes'][:, 0] - 1
            out.append(dict(r, boxes=b, flipped=True))
    return out


def make(cfg, db, backend):
    return IT.MNIteratorE2E(copy.deepcopy(db), cfg, batch_size=16, seed=7, plan_backend=backend,
                            device="cuda:0" if backend == "device" else None)


def run_config(name, cfg, db, repeats):
    its = {b: make(cfg, db, b) for b in ("host", "device")}
    assert its["host"].plan_digest == its["device"].plan_digest, name
    t = {"host": [], "device": []}
    dev = its["device"]._device_plan
    kernel, peak = [], 0
    for _ in range(repeats):
        for b in ("host", "device"):
            if b == "device":
                torch.cuda.reset_peak_memory_stats()
            host.srand(1)
            t0 = time.perf_counter()
            its[b].reset()
            t[b].append((time.perf_counter() - t0) * 1e3 / len(db))
            if b == "device":
                kernel.append(dev.stats["kernel_ms"] / len(db))
                peak = max(peak, torch.cuda.max_memory_allocated())
    assert its["host"].plan_digest == its["device"].plan_digest, name
    r = dict(config=name, images=len(db), boxes=int(dev.box_off[-1]), host_ms_per_image=[round(x, 4) for x in t["host"]],
             device_ms_per_image=[round(x, 4) for x in t["device"]],
             device_kernel_ms_per_image=[round(x, 4) for x in kernel], h2d_bytes_per_epoch=int(dev.stats["h2d_bytes"]),
             resident_device_bytes=int(dev.resident_device_bytes()), peak_device_bytes=int(peak),
             launches_per_epoch=int(dev.stats["launches"]))
    print("%-28s host %s ms/img  device %s ms/img (kernels %s)  H2D %.1f MB  resident %.1f MB  peak %.1f MB" % (
        name, r["host_ms_per_image"], r["device_ms_per_image"], r["device_kernel_ms_per_image"],
        r["h2d_bytes_per_epoch"] / 1e6, r["resident_device_bytes"] / 1e6, r["peak_device_bytes"] / 1e6), flush=True)
    return r


def replay(cfg, db, epochs=3):
    out = {}
    for b in ("host", "device"):
        t0 = time.perf_counter()
        it = make(cfg, db, b)
        for _ in range(epochs):
            it.reset()
        out[b + "_s"] = round(time.perf_counter() - t0, 3)
        out[b + "_digest"] = it.plan_digest
    assert out["host_digest"] == out["device_digest"]
    print("replay of %d epochs (+ construction), %d images: host %.3f s, device %.3f s" % (
        epochs, len(db), out["host_s"], out["device_s"]), flush=True)
    return dict(epochs=epochs, images=len(db), host_s=out["host_s"], device_s=out["device_s"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=400)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "plan_time.py measures the device plan and needs a CUDA device"
    print("card:", card())
    res = []
    for scales in ("resolution", "paper"):
        for n_prop in (0, 300, 1000):
            cfg = IT.default_config(neg=n_prop > 0)
            if scales == "paper":
                cfg.TRAIN.SCALES = load_data.PAPER_COCO_SCALES
            res.append(run_config("%s, %s" % (scales, "GT only" if n_prop == 0 else "%d proposals" % n_prop), cfg,
                                  roidb(a.images, n_prop, False), a.repeats))
    cfg = IT.default_config(neg=True)
    res.append(run_config("resolution, 300 prop, flipped", cfg, roidb(a.images // 2, 300, True), a.repeats))
    rp = replay(cfg, roidb(a.images, 1000, False))
    print(json.dumps(dict(card=card(), configs=res, replay=rp)))


if __name__ == "__main__":
    main()
