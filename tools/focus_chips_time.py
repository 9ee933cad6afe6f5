"""Times AutoFocus FocusChip generation (`chips_inference.add_chips`) on the host and on the device side by side, and
`sniper_focus_chips` alone, and prints the card's name, power limit and max SM clock next to the numbers, then one JSON
line.

  workload  seeded, COCO-val shaped: --images images of COCO's common sizes, their first-scale maps (TEST.SCALES[0],
            the whole image) and then, from the chips those give, their second-scale chip maps (TEST.SCALES[1]), as the
            pyramid feeds add_chips at the two scales that feed a pruned scale.  Random network weights give
            near-uniform FocusPixel maps, so the maps are synthetic: a low background and a few Gaussian blobs per map
            (sparse FocusPixels), stored in the `focus_map` layout (channel 1 of a [B, Hc, Wc, 2] tensor, batches of
            --batch crops).
  add_chips host `add_chips` on the maps' host copies (gmask per map) against `add_chips` on the `DeviceFocusMaps`
            (table build, one launch, the chips copied back, the area sums), alternated, host clock around work that
            ends in a synchronise; the results are compared byte for byte first.
  kernel    `sniper_focus_chips` alone on each scale's table: CUDA events over --launches launches queued behind a spin
            kernel.

    python tools/focus_chips_time.py [--images 5000] [--repeats 3] [--launches 20]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from sniper_b200 import chips_inference as CI, iterator as IT, ops  # noqa: E402
from sniper_b200._lib import check, lib  # noqa: E402

COCO_SIZES = [((640, 480), 0.45), ((480, 640), 0.15), ((640, 427), 0.15), ((427, 640), 0.05), ((500, 375), 0.05),
              ((612, 612), 0.05), ((640, 360), 0.05), ((375, 500), 0.05)]


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip().replace("\n", " | ")


def blob_map(rng, H, W, background, peak):
    y, x = np.mgrid[0:H, 0:W]
    m = rng.rand(H, W) * background
    for _ in range(rng.poisson(2.0)):
        cy, cx, s = rng.uniform(0, H), rng.uniform(0, W), rng.uniform(0.5, 2.5)
        m = np.maximum(m, peak * rng.uniform(0.5, 1.0) * np.exp(-((y - cy) ** 2 + (x - cx) ** 2) / (2 * s * s)))
    return m.astype(np.float32)


def scale_maps(roidb, scale, rng, batch, background, peak):
    """DeviceFocusMaps over every crop of roidb at `scale` (map extents as the test iterator gives them)."""
    crops = [(i, j) for i, r in enumerate(roidb) for j in range(len(r['inference_crops']))]
    maps = CI.DeviceFocusMaps([len(r['inference_crops']) for r in roidb], 16)
    for b0 in range(0, len(crops), batch):
        part = crops[b0:b0 + batch]
        info = np.zeros((len(part), 3), np.float32)
        for k, (i, j) in enumerate(part):
            r, c = roidb[i], roidb[i]['inference_crops'][j]
            s = CI.image_scale(r['width'], r['height'], scale)
            info[k] = [int(np.rint((c[3] - c[1]) * s)), int(np.rint((c[2] - c[0]) * s)), s]
        Hc, Wc = int(math.ceil(info[:, 0].max() / 16)), int(math.ceil(info[:, 1].max() / 16))
        full = np.zeros((len(part), Hc, Wc, 2), np.float32)
        for k in range(len(part)):
            H, W = int(math.ceil(info[k, 0] / 16)), int(math.ceil(info[k, 1] / 16))
            full[k, :H, :W, 1] = blob_map(rng, H, W, background, peak)
        full[..., 0] = 1 - full[..., 1]
        maps.add(torch.from_numpy(full).cuda()[..., 1], info, [i for i, _ in part], [j for _, j in part])
    return maps


def copy_db(roidb):
    return [dict(r) for r in roidb]


def time_scale(roidb, maps, scale_id, cfg, repeats):
    host_maps = [[maps[i][j] for j in range(len(maps[i]))] for i in range(len(maps))]
    db_h, db_d = copy_db(roidb), copy_db(roidb)
    a_h = CI.add_chips(db_h, host_maps, scale_id, cfg)
    a_d = CI.add_chips(db_d, maps, scale_id, cfg)
    assert np.array([a_h]).tobytes() == np.array([a_d]).tobytes()
    assert all(h['inference_crops'].tobytes() == d['inference_crops'].tobytes() for h, d in zip(db_h, db_d))
    host_s, dev_s = [], []
    for _ in range(repeats):
        t0 = time.perf_counter()
        CI.add_chips(copy_db(roidb), host_maps, scale_id, cfg)
        host_s.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        CI.add_chips(copy_db(roidb), maps, scale_id, cfg)
        torch.cuda.synchronize()
        dev_s.append(time.perf_counter() - t0)
    return db_d, a_d, host_s, dev_s


def kernel_alone(roidb, maps, scale_id, cfg, launches):
    hp = cfg.TEST.CHIP_HYPERPARAMS[scale_id]
    index, geometry = maps.focus_table(roidb, cfg.TEST.SCALES[scale_id])
    table = ops.focus_chips_table(maps.tensors, index, geometry)
    n = len(table)
    ws_off = np.zeros(n + 1, np.int64)
    L = lib()
    check(L.sniper_focus_chips_workspace_bytes(table.ctypes.data, n, ws_off.ctypes.data))
    d_table, d_ws_off = torch.from_numpy(table).cuda(), torch.from_numpy(ws_off).cuda()
    ws = torch.empty(max(int(ws_off[-1]), 1), dtype=torch.uint8, device="cuda")
    cap = 8
    chips = torch.empty(n, cap, 4, dtype=torch.float64, device="cuda")
    counts = torch.empty(n, dtype=torch.int32, device="cuda")
    thr = float(ops.focus_threshold(hp[1]))

    def launch():
        check(L.sniper_focus_chips(d_table.data_ptr(), d_ws_off.data_ptr(), table.ctypes.data, ws_off.ctypes.data, n,
                                   int(hp[0]), thr, int(hp[2]), ws.data_ptr(), cap, chips.data_ptr(), counts.data_ptr(),
                                   torch.cuda.current_stream().cuda_stream))
    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda._sleep(int(1e8))
    e0.record()
    for _ in range(launches):
        launch()
    e1.record()
    torch.cuda.synchronize()
    cells = int((table[:, 3] * table[:, 4]).sum())
    return dict(maps=n, cells=cells, largest=[int(table[:, 3].max()), int(table[:, 4].max())],
                us_per_launch=round(e0.elapsed_time(e1) * 1e3 / launches, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--batch", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("focus_chips_time.py measures on a CUDA device; none is present")
    c = card()
    print("card:", c, flush=True)
    cfg = IT.default_config()
    rng = np.random.RandomState(0)
    sizes, p = [s for s, _ in COCO_SIZES], np.array([q for _, q in COCO_SIZES])
    pick = rng.choice(len(sizes), args.images, p=p / p.sum())
    roidb = [dict(width=sizes[k][0], height=sizes[k][1], inference_crops=np.array([[0, 0, sizes[k][0], sizes[k][1]]]))
             for k in pick]
    out = dict(card=c, images=args.images, repeats=args.repeats, scales=[])
    for scale_id in (0, 1):
        hp = cfg.TEST.CHIP_HYPERPARAMS[scale_id]
        # background below the scale's threshold, blobs above it
        maps = scale_maps(roidb, cfg.TEST.SCALES[scale_id], rng, args.batch, background=0.9 * hp[1], peak=1.0)
        db_next, area, host_s, dev_s = time_scale(roidb, maps, scale_id, cfg, args.repeats)
        k = kernel_alone(roidb, maps, scale_id, cfg, args.launches)
        row = dict(scale=list(cfg.TEST.SCALES[scale_id]), hyperparams=list(hp), maps=k['maps'], cells=k['cells'],
                   largest_map=k['largest'], chips_out=int(sum(len(r['inference_crops']) for r in db_next)),
                   pixels_next_scale_pct=round(100.0 * area[0] / area[1], 2),
                   host_add_chips_s=[round(t, 4) for t in host_s], device_add_chips_s=[round(t, 4) for t in dev_s],
                   kernel_us=k['us_per_launch'])
        out['scales'].append(row)
        print("scale %s: %d maps (%d cells, largest %d x %d) -> %d chips (%.1f%% of the next scale's pixels); add_chips "
              "host %.3f s (min of %d), device %.4f s end to end; kernel alone %.1f us"
              % (row['scale'], row['maps'], row['cells'], k['largest'][0], k['largest'][1], row['chips_out'],
                 row['pixels_next_scale_pct'], min(host_s), args.repeats, min(dev_s), k['us_per_launch']), flush=True)
        roidb = db_next
        del maps
    print(json.dumps(out))


if __name__ == "__main__":
    main()
