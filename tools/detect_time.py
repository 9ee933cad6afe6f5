"""Times the AutoFocus inference pyramid (BASELINE config 5) with the host and the device detection backend side by
side, and `sniper_detect_post` alone, and prints the card's name and power limit next to the numbers, then one JSON line.

  pyramid  the workload of `bench.py --config5`: seeded synthetic 1333x800 / 800x1333 images, one training step for
           non-trivial moving statistics, `enable_autofocus`, `tester.imdb_detection_wrapper` over TEST.SCALES.  One
           warm-up pyramid per backend, then --repeats whole pyramids per backend, ALTERNATED (host, device, host, ...);
           host clock around work that ends in torch.cuda.synchronize().  Per backend: images/s (mean, min, max over the
           repeats), per-scale detect_s / post_s / total_s, aggregation seconds.  The weights are random, so the number of
           rows passing the score threshold is whatever it is; it is printed, it is the workload size.
  kernel   `ops.detect_post` alone at the three scales' batch shapes (B x 300 rois x 81 classes) on a softmax of scaled
           noise: CUDA events over --launches launches into a buffer that is rewound every launch, queued behind a
           spin kernel so that the device runs them back to back whatever the host's enqueue rate, and the algorithmic
           bytes (inputs once, emitted rows and keys once) over that time.

    python tools/detect_time.py [--images 64] [--repeats 3] [--launches 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from sniper_b200 import inference, iterator as IT, model, ops, synth_batch, tester as TS  # noqa: E402


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip().replace("\n", " | ")


def pyramid(n_images, repeats):
    cfg = IT.default_config()
    rng = np.random.RandomState(5)
    roidb = [dict(width=W, height=H, image_data=rng.randint(0, 256, (H, W, 3)).astype(np.uint8))
             for (W, H) in [((1333, 800) if rng.rand() < 0.7 else (800, 1333)) for _ in range(n_images)]]
    mc = model.Cfg()
    mc.batch_images = 2
    net = model.SniperResNet101(mc, deform_offset_std=0.01)
    net.train_step(synth_batch.make_batch(2, seed=7, device="cuda"), lr=0.001)
    net.enable_autofocus(seed=3)
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
            if 'chip_gen_s' in st[0]:
                row['chip_gen_s'] = round(float(np.mean([x['chip_gen_s'] for x in st])), 4)
            per_scale.append(row)
        agg = [r[1]['nms_s'] for r in runs[b]]
        out[b] = dict(images_per_s=round(n_images / secs.mean(), 3), images_per_s_min=round(n_images / secs.max(), 3),
                      images_per_s_max=round(n_images / secs.min(), 3), seconds=[round(float(t), 3) for t in secs],
                      aggregate_s=round(float(np.mean(agg)), 4), aggregate_s_all=[round(float(t), 4) for t in agg],
                      per_scale=per_scale, final_detections=final[b])
        print("%-6s backend: %.2f images/s (%.2f .. %.2f over %d pyramids of %d images), aggregation %.3f s, %d final "
              "detections" % (b, out[b]['images_per_s'], out[b]['images_per_s_min'], out[b]['images_per_s_max'], repeats,
                              n_images, out[b]['aggregate_s'], final[b]), flush=True)
        for row in per_scale:
            print("         scale %s: %d chips in %d batches, detect %.3f s, post %.3f s, total %.3f s%s%s"
                  % (row['scale'], row['chips'], row['batches'], row['detect_s'], row['post_s'], row['total_s'],
                     ", %d rows pass the threshold and filters" % row['detections_pre_nms']
                     if 'detections_pre_nms' in row else "",
                     ", FocusChips %.4f s" % row['chip_gen_s'] if 'chip_gen_s' in row else ""), flush=True)
    del net
    torch.cuda.empty_cache()
    return out, list(cfg.TEST.BATCH_IMAGES)


def kernel_alone(batch_sizes, launches, R=300, K=81):
    out = []
    for scale, B in enumerate(batch_sizes):
        rng = np.random.RandomState(scale)
        rois = np.zeros((B * R, 5), np.float32)
        rois[:, 0] = np.repeat(np.arange(B), R)
        xy = rng.uniform(0, 400, (B * R, 2))
        rois[:, 1:3], rois[:, 3:5] = xy, xy + rng.uniform(8, 300, (B * R, 2))
        z = rng.randn(B * R, K) * 10.0
        e = np.exp(z - z.max(1, keepdims=True))
        t = [torch.from_numpy(a).cuda() for a in (rois, (e / e.sum(1, keepdims=True)).astype(np.float32),
                                                 (rng.randn(B * R, K + 4) * 0.5).astype(np.float32))]
        deltas = t[2][:, K:K + 4]
        info = torch.tensor([[512.0, 704.0, 1.0]] * B).cuda()
        db = [dict(width=704, height=512, inference_crops=np.array([[40.0, 30.0, 600.0, 480.0]] * B))]
        chips = torch.from_numpy(inference.chip_table(db, [0] * B, list(range(B)), True, (16, 90))).cuda()
        dets = inference.DeviceDetections("cuda", capacity=B * R * (K - 1), growable=False)

        def launch():
            dets.state.zero_()
            ops.detect_post(t[0], t[1], deltas, info, chips, dets.rows, dets.keys, dets.state, dets.workspace, scale=scale)
        for _ in range(5):
            launch()
        torch.cuda.synchronize()
        n = int(dets.state[0])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(int(1e8))                          # ~50 ms: the launches below are all queued before it ends
        e0.record()
        for _ in range(launches):
            launch()
        e1.record()
        torch.cuda.synchronize()
        base0, base1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(int(1e8))
        base0.record()
        for _ in range(launches):
            dets.state.zero_()
        base1.record()
        torch.cuda.synchronize()
        us = (e0.elapsed_time(e1) - base0.elapsed_time(base1)) * 1e3 / launches
        nbytes = B * R * (5 + K + 4) * 4 + B * (3 * 4 + 12 * 8) + n * (5 * 4 + 8)
        out.append(dict(B=B, R=R, K=K, rows_emitted=n, us_per_launch=round(us, 2), algorithmic_kb=round(nbytes / 1e3, 1),
                        gb_per_s=round(nbytes / us / 1e3, 2)))
        print("kernel  B=%d x %d rois x %d classes: %d rows emitted, %.2f us per launch (mean of %d, the cursor reset "
              "subtracted), %.1f KB algorithmic -> %.2f GB/s" % (B, R, K, n, us, launches, nbytes / 1e3, nbytes / us / 1e3),
              flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--launches", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("detect_time.py measures on a CUDA device; none is present")
    assert args.images >= 1 and args.repeats >= 1 and args.launches >= 1
    c = card()
    print("card:", c, flush=True)
    pyr, batch_sizes = pyramid(args.images, args.repeats)
    print(json.dumps({"card": c, "images": args.images, "repeats": args.repeats, "pyramid": pyr,
                      "kernel": kernel_alone(batch_sizes, args.launches)}))


if __name__ == "__main__":
    main()
