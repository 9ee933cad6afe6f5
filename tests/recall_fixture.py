"""The proposal-recall cases of tests/golden/recall_ref.npz (written by oracle/run_ref_recall.py from the reference's
own IMDB.evaluate_recall), rebuilt as roidbs, plus a seeded COCO-shaped set for the sizes the file cannot hold."""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "golden", "recall_ref.npz")
CASES = ("hand", "seeded", "thr1", "thr8", "thr9", "thr130", "merged", "u16props")


def load():
    return dict(np.load(PATH))


def _split(a, n):
    return np.split(a, np.cumsum(n)[:-1]) if len(n) else []


def case(fx, name):
    """(roidb, candidate_boxes, thresholds, num_images) of a golden case."""
    k = name + '_'
    n = fx[k + 'n']
    roidb = [{'boxes': b, 'gt_classes': c, 'gt_overlaps': o}
             for b, c, o in zip(_split(fx[k + 'boxes'], n), _split(fx[k + 'gt_classes'], n),
                                _split(fx[k + 'gt_overlaps'], n))]
    cand = _split(fx[k + 'cand'], fx[k + 'cand_n']) if k + 'cand' in fx else None
    thr = fx[k + 'thresholds'] if k + 'thresholds' in fx else None
    return roidb, cand, thr, int(fx[k + 'num_images'])


def expected(fx, name):
    """(text, recalls [7, T], sorted gt_overlaps per range) of the reference."""
    k = name + '_'
    return str(fx[k + 'text']), fx[k + 'recalls'], _split(fx[k + 'ov'], fx[k + 'ov_n'])


def coco_like(seed, n_img, props=(1000, 3000), gts=7, crowded=0.01, dtype=np.float32, big=(60, 100)):
    """A seeded COCO-train-shaped set: uint16 GT roidb entries (some over 256^2 in area, some crowd rows), a few images
    with 60-100 GTs, and float32 proposals clustered around the GTs (1000-3000 per image).  Returns (roidb,
    candidate_boxes)."""
    rng = np.random.RandomState(seed)
    roidb, cand = [], []
    for i in range(n_img):
        W, H = rng.randint(400, 641), rng.randint(300, 481)
        k = rng.randint(*big) if rng.rand() < crowded else rng.poisson(gts)
        s = np.exp(rng.uniform(np.log(6), np.log(min(W, H) * 0.95), k))
        w = np.clip(s * np.exp(rng.uniform(-0.5, 0.5, k)), 2, W - 2)
        h = np.clip(s * np.exp(rng.uniform(-0.5, 0.5, k)), 2, H - 2)
        x, y = rng.uniform(0, W - w), rng.uniform(0, H - h)
        g = np.round(np.stack([x, y, x + w, y + h], 1)).astype(np.uint16)
        cls = rng.randint(1, 81, k).astype(np.int32)
        ov = np.zeros((k, 81), np.float32)
        ov[np.arange(k), cls] = np.where(rng.rand(k) < 0.03, -1.0, 1.0)
        roidb.append({'boxes': g, 'gt_classes': cls, 'gt_overlaps': ov})
        m = rng.randint(*props)
        p = np.empty((m, 4))
        near = rng.rand(m) < 0.5 if k else np.zeros(m, bool)
        src = g[rng.randint(max(k, 1), size=m) % max(k, 1)].astype(np.float64) if k else np.zeros((m, 4))
        p[near] = src[near] + rng.randn(int(near.sum()), 4) * rng.choice([1.0, 6.0, 25.0], (int(near.sum()), 1))
        far = ~near
        cx, cy = rng.uniform(0, W, far.sum()), rng.uniform(0, H, far.sum())
        sw, sh = np.exp(rng.uniform(np.log(8), np.log(400), (2, far.sum())))
        p[far] = np.stack([cx - sw / 2, cy - sh / 2, cx + sw / 2, cy + sh / 2], 1)
        p[:, 0::2] = np.clip(p[:, 0::2], 0, W - 1)
        p[:, 1::2] = np.clip(p[:, 1::2], 0, H - 1)
        p[:, 2:] = np.maximum(p[:, 2:], p[:, :2])
        cand.append(p.astype(dtype))
    return roidb, cand
