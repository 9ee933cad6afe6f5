"""Times the negative-chip proposal pipeline and prints the card's name and power limit next to the numbers, then one
JSON line:

  extraction  MNIteratorTest + Tester.extract_proposals (forward_rpn) per TEST scale at the reference's scales and batch
              sizes (1400x2000 / 2, 800x1280 / 2, 480x512 / 4) on synthetic 1333x800 images (TF32 backbone); device
              events around the whole pass after one warm-up batch, pixels and host post-processing included.
  loading     the NMS pass of proposals.IMDB.load_rpn_data over --load-images images of 900 rows (three scales x 300):
              the device path (proposals.nms_keeps: H2D, one launch per 4096 images, D2H; host clock after a
              synchronise) and the kernels alone (device events), against the numpy restatement of nmsp on the host,
              timed on the first --host-images images.  The keep lists of those images are compared.

    python tools/proposal_time.py [--images 16] [--load-images 20000] [--host-images 200]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import proposal_nms_np as PN  # noqa: E402
from sniper_b200 import iterator as IT  # noqa: E402
from sniper_b200 import model, ops, proposals, tester  # noqa: E402

TEST_SCALES = [((1400, 2000), 2), ((800, 1280), 2), ((480, 512), 4)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=10).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def extraction(n_images):
    cfg = IT.default_config()
    mc = model.Cfg()
    mc.batch_images = 2
    net = model.SniperResNet101(mc, device="cuda:0", seed=5)
    db = IT.synthetic_roidb(n_images, seed=1, n_prop=0)
    out = {}
    for scale, nbatch in TEST_SCALES:
        warm = tester.MNIteratorTest(db[:nbatch], cfg, scale, batch_size=nbatch)
        tester.Tester(net, None, db[:nbatch], warm, cfg, batch_size=nbatch, num_classes=1).extract_proposals()
        it = tester.MNIteratorTest(db, cfg, scale, batch_size=nbatch)
        t = tester.Tester(net, None, db, it, cfg, batch_size=nbatch, num_classes=1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        t.extract_proposals()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        out["%dx%d" % scale] = dict(batch=nbatch, images=it.size, ms=round(ms, 1), images_per_s=round(it.size * 1e3 / ms, 1))
        print("extraction %dx%d / %d: %d images (padded batches) in %.1f ms -> %.1f images/s"
              % (scale[0], scale[1], nbatch, it.size, ms, it.size * 1e3 / ms), flush=True)
    del net
    torch.cuda.empty_cache()
    return out


def proposal_lists(n, rng):
    """n images of 900 rows: three 300-row scales of clustered boxes over a 1333x800 image, distinct scores."""
    out = []
    for _ in range(n):
        k = 60
        cx, cy = rng.uniform(0, 1333, k), rng.uniform(0, 800, k)
        s = np.exp(rng.uniform(np.log(16), np.log(400), k))
        j = rng.randint(0, k, 900)
        w, h = s[j] * np.exp(rng.randn(900) * 0.15), s[j] * np.exp(rng.randn(900) * 0.15)
        x, y = cx[j] + rng.randn(900) * 0.1 * s[j], cy[j] + rng.randn(900) * 0.1 * s[j]
        d = np.stack([np.clip(x - w / 2, 0, 1332), np.clip(y - h / 2, 0, 799), np.clip(x + w / 2, 0, 1332),
                      np.clip(y + h / 2, 0, 799), rng.permutation(900) / 900.0 + 1e-3], 1).astype(np.float32)
        out.append(d)
    return out


def loading(n_images, n_host):
    rng = np.random.RandomState(0)
    lists = proposal_lists(n_images, rng)
    proposals.nms_keeps(lists[:64])                         # module load, allocator warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    keeps = proposals.nms_keeps(lists)
    torch.cuda.synchronize()
    dev_s = time.perf_counter() - t0
    # the kernels alone: every chunk uploaded first, device events around the launches
    chunks = []
    for c0 in range(0, n_images, proposals.NMS_CHUNK):
        part = lists[c0:c0 + proposals.NMS_CHUNK]
        off = np.concatenate([[0], np.cumsum([len(p) for p in part])]).astype(np.int32)
        chunks.append((torch.from_numpy(np.concatenate(part)).cuda(), off, torch.from_numpy(off).cuda(),
                       torch.empty(len(part), dtype=torch.int32, device="cuda"),
                       torch.empty(int(off[-1]), dtype=torch.int32, device="cuda")))
    lib = ops.lib()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for dets, off, off_dev, counts, keep in chunks:
        ops.check(lib.sniper_proposal_nms_batched(dets.data_ptr(), off_dev.data_ptr(), off.ctypes.data, len(off) - 1,
                                                  counts.data_ptr(), keep.data_ptr(), ops._stream()))
    e1.record()
    torch.cuda.synchronize()
    kernel_ms = e0.elapsed_time(e1)
    t0 = time.perf_counter()
    host = [PN.nmsp_keep(d) for d in lists[:n_host]]
    host_s = time.perf_counter() - t0
    same = all(np.array_equal(a, b) for a, b in zip(host, keeps[:n_host]))
    kept = float(np.mean([len(k) for k in keeps]))
    res = dict(images=n_images, rows_per_image=900, mean_kept=round(kept, 1), device_pass_s=round(dev_s, 3),
               kernels_ms=round(kernel_ms, 1), host_images=n_host, host_ms_per_image=round(host_s * 1e3 / n_host, 2),
               host_keeps_equal=same)
    print("loading NMS, %d images x 900 rows (mean %.1f kept): device pass %.3f s (kernels %.1f ms); numpy restatement "
          "%.2f ms/image on the host (%d images timed); keep lists equal: %s"
          % (n_images, kept, dev_s, kernel_ms, host_s * 1e3 / n_host, n_host, same), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--load-images", type=int, default=20000)
    ap.add_argument("--host-images", type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "proposal_time.py measures on a CUDA device"
    print("card:", card(), flush=True)
    result = {"card": card(), "extraction": extraction(args.images),
              "loading": loading(args.load_images, args.host_images)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
