"""Times the MobileNetV2 multi-scale inference pyramid (BASELINE config 4's test block) with the host and the device
detection backend side by side, and prints the card's name, power limit and maximum SM clock next to the numbers, then
one JSON line.

  Seeded synthetic 1333x800 / 800x1333 images, a bf16 `SniperMobileNetV2` with random weights after one training step
  (non-trivial moving statistics), `tester.imdb_detection_wrapper` over TEST.SCALES of
  `iterator.default_config(network="mobilenetv2")`: (1400,2000) / (800,1280) / (480,512), batches 2 / 2 / 4.  One
  warm-up pyramid per backend, then --repeats whole pyramids per backend, ALTERNATED (host, device, host, ...); host
  clock around work that ends in torch.cuda.synchronize().  Per backend: images/s (mean, min, max over the repeats),
  per-scale detect_s / post_s / total_s, aggregation seconds.  The weights are random, so the number of rows passing
  the score threshold is whatever it is; it is printed, it is the workload size.

    python tools/mnv2_detect_time.py [--images 128] [--repeats 3]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from sniper_b200 import iterator as IT, model_mnv2, synth_batch, tester as TS  # noqa: E402
from detect_time import card  # noqa: E402


def pyramid(n_images, repeats):
    cfg = IT.default_config(network="mobilenetv2")
    rng = np.random.RandomState(5)
    roidb = [dict(width=W, height=H, image_data=rng.randint(0, 256, (H, W, 3)).astype(np.uint8))
             for (W, H) in [((1333, 800) if rng.rand() < 0.7 else (800, 1333)) for _ in range(n_images)]]
    mc = model_mnv2.MCfg()
    mc.batch_images, mc.bf16 = 2, True
    net = model_mnv2.SniperMobileNetV2(mc, device="cuda", seed=3)
    net.train_step(synth_batch.make_batch(2, seed=7, device="cuda", A=mc.num_anchors, stride=mc.feat_stride), lr=0.001)
    backends = ("host", "device")
    final = {}
    for b in backends:                                       # warm-up: allocator, lazy kernel loading, pinned pools
        boxes, _ = TS.imdb_detection_wrapper(net, cfg, roidb, detect_backend=b)
        final[b] = int(sum(len(boxes[j][i]) for j in range(1, 81) for i in range(n_images)))
    torch.cuda.synchronize()
    runs = {b: [] for b in backends}
    for _ in range(repeats):
        for b in backends:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, stats = TS.imdb_detection_wrapper(net, cfg, roidb, detect_backend=b)
            torch.cuda.synchronize()
            runs[b].append((time.perf_counter() - t0, stats))
    out = {}
    for b in backends:
        secs = np.array([t for t, _ in runs[b]])
        per_scale = []
        for s in range(len(cfg.TEST.SCALES)):
            st = [r[1]['scales'][s] for r in runs[b]]
            row = dict(scale=list(st[0]['scale']), chips=st[0]['chips'], batches=st[0]['batches'])
            for k in ("detect_s", "post_s", "total_s"):
                row[k] = round(float(np.mean([x[k] for x in st])), 4)
            if 'detections_pre_nms' in st[0]:
                row['detections_pre_nms'] = st[0]['detections_pre_nms']
            per_scale.append(row)
        agg = [r[1]['nms_s'] for r in runs[b]]
        out[b] = dict(images_per_s=round(n_images / secs.mean(), 3), images_per_s_min=round(n_images / secs.max(), 3),
                      images_per_s_max=round(n_images / secs.min(), 3), seconds=[round(float(t), 3) for t in secs],
                      aggregate_s=round(float(np.mean(agg)), 4), per_scale=per_scale, final_detections=final[b])
        print("%-6s backend: %.2f images/s (%.2f .. %.2f over %d pyramids of %d images), aggregation %.3f s, %d final "
              "detections" % (b, out[b]['images_per_s'], out[b]['images_per_s_min'], out[b]['images_per_s_max'], repeats,
                              n_images, out[b]['aggregate_s'], final[b]), flush=True)
        for row in per_scale:
            print("         scale %s: %d chips in %d batches, detect %.3f s, post %.3f s, total %.3f s%s"
                  % (row['scale'], row['chips'], row['batches'], row['detect_s'], row['post_s'], row['total_s'],
                     ", %d rows pass the threshold and filters" % row['detections_pre_nms']
                     if 'detections_pre_nms' in row else ""), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mnv2_detect_time.py measures on a CUDA device; none is present")
    assert args.images >= 1 and args.repeats >= 1
    c = card()
    print("card:", c, flush=True)
    print(json.dumps({"card": c, "images": args.images, "repeats": args.repeats,
                      "pyramid": pyramid(args.images, args.repeats)}))


if __name__ == "__main__":
    main()
