"""Times TEST.CONCURRENT_JOBS: images/s of tester.imdb_detection_wrapper (AutoFocus pyramid of iterator.default_config,
device detection back end) and of tester.imdb_proposal_extraction_wrapper (the config's three test scales) on --images
synthetic 1333x800 COCO-shaped images (TF32 ResNet-101 of seed 5), and prints the card's name and power limit next to
the numbers, then one JSON line.

  one GPU    concurrent_jobs 1 against 2 in one process, alternated --reps times after a warm-up run of each: the
             cost of the second job's partial batches.  Host clock around the wrapper call, which ends in a device
             synchronise (the soft-NMS result, the proposals' copy to the host).
  two GPUs   (when two are visible) the same wrappers with 2 jobs on one rank against 2 ranks (this script under
             torch.distributed.run, NCCL, one GPU each, started with --ranks); the two-rank time is rank 0's, from
             before the roidb check to the merged result.

    python tools/concurrent_test_time.py [--images 32] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from sniper_b200 import iterator as IT  # noqa: E402
from sniper_b200 import model, tester  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=10).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def make(device):
    cfg = IT.default_config()
    mc = model.Cfg()
    mc.batch_images = 2
    net = model.SniperResNet101(mc, device=device, seed=5)
    net.enable_autofocus(seed=3)
    return cfg, net


def one_run(kind, net, cfg, db, jobs, device, group=None):
    """Seconds of one wrapper call over `db` (fresh entries, so every run starts from the full-image chips)."""
    db = [dict(r) for r in db]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if kind == "detect":
        tester.imdb_detection_wrapper(net, cfg, db, device=device, detect_backend="device", concurrent_jobs=jobs,
                                      group=group)
    else:
        with tempfile.TemporaryDirectory() as d:
            cfg.dataset.test_image_set = "timing"
            tester.imdb_proposal_extraction_wrapper(net, cfg, db, d, device=device, concurrent_jobs=jobs, group=group)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def one_gpu(n_images, reps):
    cfg, net = make("cuda:0")
    db = IT.synthetic_roidb(n_images, seed=1, n_prop=0)
    out = {}
    for kind in ("detect", "proposals"):
        for jobs in (1, 2):
            one_run(kind, net, cfg, db[:4], jobs, "cuda:0")                    # warm-up
        times = {1: [], 2: []}
        for _ in range(reps):
            for jobs in (1, 2):
                times[jobs].append(one_run(kind, net, cfg, db, jobs, "cuda:0"))
        out[kind] = {"jobs%d" % j: dict(s=[round(t, 3) for t in ts], images_per_s=round(n_images / np.median(ts), 2))
                     for j, ts in times.items()}
        print("%-9s %d images, one GPU: 1 job %.2f images/s, 2 jobs %.2f images/s (median of %d, alternated)"
              % (kind, n_images, out[kind]["jobs1"]["images_per_s"], out[kind]["jobs2"]["images_per_s"], reps),
              flush=True)
    del net
    torch.cuda.empty_cache()
    return out


def ranks(n_images, reps):
    """Under torch.distributed.run: every rank on cuda:LOCAL_RANK, 2 jobs per wrapper call; rank 0 prints a JSON line."""
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist = torch.distributed
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = "cuda:%d" % local
    cfg, net = make(dev)
    db = IT.synthetic_roidb(n_images, seed=1, n_prop=0)
    out = {}
    try:
        for kind in ("detect", "proposals"):
            one_run(kind, net, cfg, db[:4], 2, dev, dist.group.WORLD)
            ts = []
            for _ in range(reps):
                dist.barrier()
                ts.append(one_run(kind, net, cfg, db, 2, dev, dist.group.WORLD))
            out[kind] = dict(s=[round(t, 3) for t in ts], images_per_s=round(n_images / np.median(ts), 2))
        if dist.get_rank() == 0:
            print("RANKS " + json.dumps(out), flush=True)
    finally:
        dist.destroy_process_group()


def two_gpus(n_images, reps):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29571", os.path.abspath(__file__), "--ranks", "--images", str(n_images),
           "--reps", str(reps)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3600, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError("the two-rank run failed:\n" + r.stdout[-3000:] + r.stderr[-5000:])
    line = [l for l in r.stdout.splitlines() if l.startswith("RANKS ")][-1]
    out = json.loads(line[len("RANKS "):])
    for kind, v in out.items():
        print("%-9s %d images, 2 jobs on 2 ranks (one GPU each): %.2f images/s" % (kind, n_images, v["images_per_s"]),
              flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ranks", action="store_true", help="(internal) one rank of the two-GPU measurement")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "concurrent_test_time.py measures on a CUDA device"
    if args.ranks:
        return ranks(args.images, args.reps)
    print("card:", card(), flush=True)
    result = {"card": card(), "images": args.images, "one_gpu": one_gpu(args.images, args.reps)}
    if torch.cuda.device_count() >= 2:
        result["two_ranks"] = two_gpus(args.images, args.reps)
    else:
        result["two_ranks"] = "not measured: one GPU visible"
        print("two ranks: not measured, one GPU visible", flush=True)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
