"""Times the COCO box evaluation on a seeded val2017-shaped synthetic set (5000 images, 80 categories, ~7 GTs and 100
detections per image) and prints the card's name and power limit next to the numbers, then one JSON line:

  device      sniper_coco_match, then the category sort + sniper_coco_accumulate, with CUDA events around the launches,
              after a warm-up, averaged over --reps runs (the CSR already on the device).
  end to end  coco.evaluate_detections(all_boxes) wall time, split into the results json writing, loadRes (json read),
              the host CSR packing and the device evaluate / accumulate (each ending in a synchronise).
  numpy       oracle/cocoeval_np.py (the float64 restatement) on this host, same CSR; its arrays are compared with the
              device's.

    python tools/cocoeval_time.py [--images 5000] [--reps 20]
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
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import cocoeval_fixture as F  # noqa: E402
import cocoeval_np  # noqa: E402
from sniper_b200 import coco, cocoeval, ops  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=10).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "cocoeval_time needs a CUDA device"
    gt, res = F.synthetic_set(7, n_img=a.images)
    out = dict(images=a.images, gts=len(gt['annotations']), detections=len(res), card=card())

    # the detector output all_boxes[class][image] that writes these results (x2 = x + w - 1)
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "data", "annotations"))
        with open(os.path.join(tmp, "data", "annotations", "instances_val2017.json"), "w") as f:
            json.dump(gt, f)
        imdb = coco.coco("val2017", tmp, os.path.join(tmp, "data"))
        img_ind = {i: k for k, i in enumerate(imdb.image_set_index)}
        cls_ind = {imdb._class_to_coco_ind[c]: k for k, c in enumerate(imdb.classes) if k}
        rows = np.array([[img_ind[r['image_id']], cls_ind[r['category_id']]] + r['bbox'] + [r['score']] for r in res])
        all_boxes = [[np.zeros((0, 5), np.float32) for _ in imdb.image_set_index] for _ in imdb.classes]
        rows = rows[np.lexsort((rows[:, 0], rows[:, 1]))]       # stable: each image keeps its results order
        keys = rows[:, 1].astype(np.int64) * len(imdb.image_set_index) + rows[:, 0].astype(np.int64)
        starts = np.flatnonzero(np.r_[True, keys[1:] != keys[:-1]])
        for s, e in zip(starts, np.r_[starts[1:], len(rows)]):
            b = rows[s:e, 2:]
            all_boxes[int(rows[s, 1])][int(rows[s, 0])] = np.stack(
                [b[:, 0], b[:, 1], b[:, 0] + b[:, 2] - 1, b[:, 1] + b[:, 3] - 1, b[:, 4]], 1).astype(np.float32)
        imdb.evaluate_detections(all_boxes)           # warm-up (module load, allocator)
        t0 = time.time()
        stats = imdb.evaluate_detections(all_boxes)
        out['end_to_end_s'] = time.time() - t0
        out['end_to_end_split_s'] = imdb.eval_times
        out['stats'] = np.asarray(stats).tolist()

    cg = cocoeval.COCO(gt)
    cd = cg.loadRes(res)
    E = cocoeval.COCOeval(cg, cd)
    E.evaluate()
    E.accumulate()
    p, pk, dv = E.params, E._pk, E._dev
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]

    def device_pass():
        ev[0].record()
        m = E._run_match(full=False)
        ev[1].record()
        order = ops.coco_category_order(dv['dt_score'], dv['dt_cat'])
        pr, rc = ops.coco_accumulate(m['dt_flags'], dv['dt_rank'], order, pk['dt_off'], m['npig'], pk['cat_pair_off'],
                                     p.maxDets, np.asarray(p.recThrs, np.float64))
        ev[2].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), pr, rc

    for _ in range(3):
        device_pass()
    t_m, t_a = [], []
    for _ in range(a.reps):
        m_ms, a_ms, pr, rc = device_pass()
        t_m.append(m_ms)
        t_a.append(a_ms)
    out['device_match_ms'] = float(np.mean(t_m))
    out['device_accumulate_ms'] = float(np.mean(t_a))
    out['device_total_ms'] = out['device_match_ms'] + out['device_accumulate_ms']

    t0 = time.time()
    r = cocoeval_np.match(pk, p.iouThrs, p.areaRng)
    t1 = time.time()
    prec, rec = cocoeval_np.accumulate(pk, r, p.maxDets, p.recThrs, pk['K'])
    out['numpy_match_s'], out['numpy_accumulate_s'] = t1 - t0, time.time() - t1
    out['equal_to_numpy'] = bool(prec.tobytes() == pr.cpu().numpy().tobytes()
                                 and rec.tobytes() == rc.cpu().numpy().tobytes())
    print("card: %s" % out['card'])
    print("device evaluate %.2f ms + accumulate %.2f ms; end to end %.2f s %s; numpy %.2f s + %.2f s; equal %s" % (
        out['device_match_ms'], out['device_accumulate_ms'], out['end_to_end_s'],
        {k: round(v, 3) for k, v in out['end_to_end_split_s'].items()}, out['numpy_match_s'],
        out['numpy_accumulate_s'], out['equal_to_numpy']))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
