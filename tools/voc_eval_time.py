"""Times the PASCAL VOC evaluation on a seeded VOC2007-test-shaped synthetic devkit (4952 images, 20 classes, ~3 objects
per image, 15% of them difficult, 200 detections per image) and prints the card's name and power limit next to the
numbers, then one JSON line:

  device      sniper_voc_match (both overlap thresholds) and sniper_voc_accumulate (11-point and area metric), with
              CUDA events around the launches, after a warm-up, averaged over --reps runs (the inputs already on the
              device).
  end to end  PascalVOC.evaluate_detections(all_boxes) wall time, split into writing the comp4 files, parsing them
              (and the annotations: the first call parses the XML, the second reads the cache), the host
              np.argsort and the device (copies included).  The second call is reported; the first call's parse too.
  numpy       oracle/voc_eval_np.py's per-detection loop and accumulation (the reference's loop, float64) on this host,
              same inputs; its arrays are compared with the device's.

    python tools/voc_eval_time.py [--images 4952] [--reps 20]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

import voc_eval_np  # noqa: E402
from sniper_b200 import _lib, pascal_voc  # noqa: E402

CLASSES = list(pascal_voc.CLASSES[1:])


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=10).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def devkit(root, n_img, seed=0, per_img=3, det_per_img=200):
    """Writes VOCdevkit/VOC2007 (annotations, image set 'test', empty JPEG files); returns (devkit, all_boxes)."""
    rng = np.random.RandomState(seed)
    vp = os.path.join(root, "VOCdevkit", "VOC2007")
    for sub in ("Annotations", os.path.join("ImageSets", "Main"), "JPEGImages"):
        os.makedirs(os.path.join(vp, sub))
    names = ["%06d" % (2 * i + 1) for i in range(n_img)]
    with open(os.path.join(vp, "ImageSets", "Main", "test.txt"), "w") as f:
        f.write("".join(n + "\n" for n in names))
    all_boxes = [[np.zeros((0, 5), np.float32) for _ in range(n_img)] for _ in range(21)]
    for i, n in enumerate(names):
        W, H = rng.randint(300, 500), rng.randint(300, 500)
        k = rng.poisson(per_img)
        c = rng.randint(20, size=k)
        wh = rng.randint(10, W // 2, (k, 2))
        xy = rng.randint(1, W // 2, (k, 2))
        g = np.concatenate([xy, xy + wh], 1)
        diff = rng.rand(k) < 0.15
        obj = "".join("<object><name>%s</name><difficult>%d</difficult><bndbox><xmin>%d</xmin><ymin>%d</ymin>"
                      "<xmax>%d</xmax><ymax>%d</ymax></bndbox></object>" % ((CLASSES[c[j]], diff[j]) + tuple(g[j]))
                      for j in range(k))
        with open(os.path.join(vp, "Annotations", n + ".xml"), "w") as f:
            f.write("<annotation><size><width>%d</width><height>%d</height></size>%s</annotation>" % (W, H, obj))
        open(os.path.join(vp, "JPEGImages", n + ".jpg"), "w").close()
        near = (rng.rand(det_per_img) < 0.5) & (k > 0)
        pick = rng.randint(max(k, 1), size=det_per_img)
        dc = np.where(near, c[pick] if k else 0, rng.randint(20, size=det_per_img))
        b = rng.uniform(0, 300, (det_per_img, 4))
        b[:, 2:] = b[:, :2] + rng.uniform(5, 150, (det_per_img, 2))
        if k:
            b = np.where(near[:, None], g[pick] - 1 + rng.randn(det_per_img, 4) * 6, b)
        d = np.concatenate([b, rng.rand(det_per_img, 1)], 1).astype(np.float32)
        for cc in range(20):
            all_boxes[cc + 1][i] = d[dc == cc]
    return os.path.join(root, "VOCdevkit"), all_boxes


def stage(imdb):
    """The device inputs voc_eval_classes builds, from the files the imdb wrote."""
    images = list(imdb.image_set_index)
    recs = {n: pascal_voc.parse_voc_rec(os.path.join(imdb.data_path, "Annotations", n + ".xml")) for n in images}
    gt_box, gt_diff, gt_off, npos = pascal_voc.gt_csr(recs, images, CLASSES)
    index = {n: i for i, n in enumerate(images)}
    boxes, pairs, det_off = [], [], [0]
    for c, cls in enumerate(CLASSES):
        ids, conf, bbox = pascal_voc.read_detections(imdb.get_result_file_template().format(cls))
        s = np.argsort(-conf)
        boxes.append(bbox[s].reshape(-1, 4))
        pairs.append(c * len(images) + np.array([index[x] for x in ids], np.int64)[s])
        det_off.append(det_off[-1] + len(s))
    return (np.concatenate(boxes), np.concatenate(pairs), gt_box, gt_diff, gt_off, npos,
            np.asarray(det_off, np.int32))


def device_time(inputs, reps):
    det_box, det_pair, gt_box, gt_diff, gt_off, npos, det_off = inputs
    dev = torch.device("cuda")
    P, N, G, C, T = gt_off.size - 1, len(det_pair), int(gt_off[-1]), len(CLASSES), 2
    pos = np.argsort(det_pair, kind="stable").astype(np.int32)
    pair_off = np.zeros(P + 1, np.int32)
    np.cumsum(np.bincount(det_pair, minlength=P), out=pair_off[1:])
    thr = np.array([0.5, 0.7])
    t07 = np.arange(0., 1.1, 0.1)
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in dict(
        box=det_box, pair_off=pair_off, pos=pos, gt_box=gt_box, gt_diff=gt_diff, gt_off=gt_off, npos=npos,
        det_off=det_off).items()}
    flags = torch.empty(T, N, dtype=torch.uint8, device=dev)
    taken = torch.empty(T, G, dtype=torch.uint8, device=dev)
    rec, prec = (torch.empty(T, N, dtype=torch.float64, device=dev) for _ in range(2))
    ap = {m: torch.empty(T, C, dtype=torch.float64, device=dev) for m in (0, 1)}
    terms = torch.empty(T, N + C, dtype=torch.float64, device=dev)
    L, s = _lib.lib(), torch.cuda.current_stream().cuda_stream

    def match():
        _lib.check(L.sniper_voc_match(d["box"].data_ptr(), d["pair_off"].data_ptr(), d["pos"].data_ptr(),
                                      d["gt_box"].data_ptr(), d["gt_diff"].data_ptr(), d["gt_off"].data_ptr(),
                                      pair_off.ctypes.data, gt_off.ctypes.data, P, thr.ctypes.data, T,
                                      flags.data_ptr(), taken.data_ptr(), s))

    def acc(m):
        _lib.check(L.sniper_voc_accumulate(flags.data_ptr(), d["det_off"].data_ptr(), d["npos"].data_ptr(),
                                           det_off.ctypes.data, C, T, m, t07.ctypes.data, t07.size, rec.data_ptr(),
                                           prec.data_ptr(), ap[m].data_ptr(), terms.data_ptr(), s))
    out = {}
    for name, fn in (("match_ms", match), ("accumulate_07_ms", lambda: acc(1)), ("accumulate_area_ms", lambda: acc(0))):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out[name] = e0.elapsed_time(e1) / reps
    res = dict(flags=flags.cpu().numpy(), rec=rec.cpu().numpy(), prec=prec.cpu().numpy(),
               ap07=ap[1].cpu().numpy(), ap=ap[0].cpu().numpy())
    return out, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4952)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("voc_eval_time: no CUDA device")
    print("card:", card())
    with tempfile.TemporaryDirectory() as root:
        dk, all_boxes = devkit(root, a.images)
        imdb = pascal_voc.PascalVOC("2007_test", root, dk)
        imdb.evaluate_detections(all_boxes)
        first = dict(imdb.eval_times)
        t0 = time.time()
        info = imdb.evaluate_detections(all_boxes)
        wall = time.time() - t0
        second = dict(imdb.eval_times)
        inputs = stage(imdb)
    n_det, n_gt = len(inputs[1]), int(inputs[4][-1])
    dev, res = device_time(inputs, a.reps)
    t0 = time.time()
    flags = voc_eval_np.match(*inputs[:5], (0.5, 0.7))
    t_match = time.time() - t0
    t0 = time.time()
    r07 = voc_eval_np.accumulate(flags, inputs[6], inputs[5], True)
    rar = voc_eval_np.accumulate(flags, inputs[6], inputs[5], False)
    t_acc = time.time() - t0
    equal = bool(flags.tobytes() == res["flags"].tobytes() and rar[0].tobytes() == res["rec"].tobytes()
                 and rar[1].tobytes() == res["prec"].tobytes() and rar[2].tobytes() == res["ap"].tobytes()
                 and r07[2].tobytes() == res["ap07"].tobytes())
    print(info.split("\n")[21], "|", info.split("\n")[-1])
    out = dict(images=a.images, classes=20, gts=n_gt, detections=n_det, device=dev,
               evaluate_detections=dict(wall_s=wall, **{k: second[k] for k in ("write_s", "parse_s", "sort_s", "device_s")},
                                        first_parse_s=first["parse_s"]),
               numpy=dict(match_s=t_match, accumulate_both_metrics_s=t_acc), numpy_equals_device=equal)
    print(json.dumps(out))
    return 0 if equal else 1


if __name__ == "__main__":
    sys.exit(main())
