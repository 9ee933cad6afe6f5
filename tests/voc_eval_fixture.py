"""tests/golden/voc_eval_ref.npz (oracle/run_ref_voc_eval.py): the reference's PASCAL VOC evaluation on synthetic
VOCdevkits.  Helpers rebuild a case's devkit and all_boxes and the device inputs (detections in the recorded order, the
GT CSR) from the recorded comp4 text."""
import os

import numpy as np

from sniper_b200 import pascal_voc

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "golden", "voc_eval_ref.npz")
CASES = ("hand", "ties07", "ties12")
CLASSES = list(pascal_voc.CLASSES[1:])


def load():
    return dict(np.load(PATH))


def write_devkit(fx, name, root, images=True):
    """VOCdevkit/VOC<year> with the case's annotations, image set 'test' and (empty) JPEG files; returns the devkit."""
    year = str(fx[name + "_year"])
    dk = os.path.join(root, "VOCdevkit")
    vp = os.path.join(dk, "VOC" + year)
    for sub in ("Annotations", os.path.join("ImageSets", "Main"), "JPEGImages"):
        os.makedirs(os.path.join(vp, sub), exist_ok=True)
    names = [str(n) for n in fx[name + "_images"]]
    with open(os.path.join(vp, "ImageSets", "Main", "test.txt"), "w") as f:
        f.write("".join(n + "\n" for n in names))
    for n, x in zip(names, fx[name + "_xml"]):
        with open(os.path.join(vp, "Annotations", n + ".xml"), "w") as f:
            f.write(str(x))
        if images:
            open(os.path.join(vp, "JPEGImages", n + ".jpg"), "w").close()
    return dk


def all_boxes(fx, name, dtype=np.float32):
    """all_boxes[21][num_images] of the case, rows in the recorded order."""
    n_img = len(fx[name + "_images"])
    d = fx[name + "_dets"]
    ab = [[np.zeros((0, 5), dtype) for _ in range(n_img)] for _ in range(21)]
    for c in range(1, 21):
        for i in range(n_img):
            sel = (d[:, 0] == c) & (d[:, 1] == i)
            if sel.any():
                ab[c][i] = d[sel, 2:].astype(np.float32).astype(dtype)
    return ab


def device_inputs(fx, name, dk):
    """(det_box [N, 4] float64, det_pair [N], gt_box, gt_difficult, gt_off, npos, det_off) in the recorded order,
    from the recorded comp4 text and the devkit's annotations."""
    year = str(fx[name + "_year"])
    images = [str(n) for n in fx[name + "_images"]]
    recs = {n: pascal_voc.parse_voc_rec(os.path.join(dk, "VOC" + year, "Annotations", n + ".xml")) for n in images}
    gt_box, gt_diff, gt_off, npos = pascal_voc.gt_csr(recs, images, CLASSES)
    index = {n: i for i, n in enumerate(images)}
    off, si = fx[name + "_det_off"], fx[name + "_sorted_inds"]
    boxes, pairs = [], []
    for c, text in enumerate(fx[name + "_text"]):
        tok = str(text).split()
        a = np.array(tok, dtype=object).reshape(-1, 6)
        s = si[off[c]:off[c + 1]]
        boxes.append(a[:, 2:].astype(np.float64)[s])
        pairs.append(c * len(images) + np.array([index[x] for x in a[:, 0]], np.int64)[s])
    return (np.concatenate(boxes).reshape(-1, 4), np.concatenate(pairs), gt_box, gt_diff, gt_off, npos,
            off.astype(np.int32))


def same(a, b):
    """Equal bytes, except that NaNs only have to sit at the same places (their sign and payload are not part of what
    the reference computes)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool((na == nb).all()) and a[~na].tobytes() == b[~nb].tobytes()
