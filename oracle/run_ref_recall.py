"""TEST INFRASTRUCTURE ONLY.  Runs the reference's OWN IMDB.evaluate_recall (lib/dataset/imdb.py:291-397) in THIS
container and writes tests/golden/recall_ref.npz (run: python oracle/build_ref_cython.py, then
python oracle/run_ref_recall.py).

imdb.py is read as text from /root/reference and executed in memory (nothing is copied into the repo).  It is Python 2,
so the print statements become calls, np.float becomes np.float64, and the imports the method does not reach (cPickle,
PIL, nms, multiprocessing) are dropped.  bbox_overlaps is the reference's bbox.pyx, cythonized into oracle/_ref/ by
build_ref_cython.py.  The module's numpy is a proxy that keeps every np.sort result (each range's sorted gt_overlaps)
and every np.zeros_like result (each range's recalls, filled in place), so both are captured at full precision.

Each case stores its roidb (boxes / gt_classes / gt_overlaps concatenated with per-image counts), its candidate_boxes,
thresholds and num_images (when given), the returned string, the recalls [7, T] and the sorted gt_overlaps."""
import contextlib
import io
import os
import re
import sys
import types

import numpy as np

REF = "/root/reference/lib/dataset"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "tests", "golden", "recall_ref.npz")
DROP = ('import cPickle', 'from PIL import Image', 'from bbox.bbox_transform import', 'from nms.nms import',
        'from multiprocessing import')
C = 5  # classes of the synthetic roidbs (background included)


def _py3(src):
    src = '\n'.join('' if l.strip().startswith(DROP) else l for l in src.split('\n'))
    src = re.sub(r'^(\s*)print (.+)$', r'\1print(\2)', src, flags=re.M)
    return re.sub(r'\bnp\.float\b', 'np.float64', src)


class _RecordingNumpy(types.ModuleType):
    """numpy, with every sort and zeros_like result kept."""
    def __init__(self):
        super().__init__("numpy")
        self.sorts, self.recalls = [], []

    def __getattr__(self, k):
        return getattr(np, k)

    def sort(self, *a, **kw):
        r = np.sort(*a, **kw)
        self.sorts.append(r)
        return r

    def zeros_like(self, *a, **kw):
        r = np.zeros_like(*a, **kw)
        self.recalls.append(r)
        return r


def load_reference():
    sys.path.insert(0, os.path.join(HERE, "_ref"))
    import ref_bbox
    ns = {"__name__": "ref_imdb", "bbox_overlaps": ref_bbox.bbox_overlaps_cython}
    exec(compile(_py3(open(os.path.join(REF, "imdb.py")).read()), "imdb.py", "exec"), ns)
    ns["np"] = _RecordingNumpy()
    return ns["IMDB"], ns["np"]


# --------------------------------------------------------------------------------------------------------------------
# roidbs: gt_roidb-like entries (uint16 boxes, int32 classes, float32 [n, C] gt_overlaps)
# --------------------------------------------------------------------------------------------------------------------
def entry(gt, cls, ovmax=None, extra=None, dtype=np.uint16):
    """gt: [k, 4] boxes; cls: classes (0 = a proposal row); ovmax: each row's gt_overlaps value (default 1 for a GT,
    0 for a proposal); extra: [j, 4] proposal rows appended with class 0."""
    gt = np.asarray(gt, np.float64).reshape(-1, 4)
    cls = np.asarray(cls, np.int32).reshape(-1)
    ov = np.where(cls > 0, 1.0, 0.0) if ovmax is None else np.asarray(ovmax, np.float64)
    if extra is not None:
        extra = np.asarray(extra, np.float64).reshape(-1, 4)
        gt = np.vstack([gt, extra])
        cls = np.concatenate([cls, np.zeros(len(extra), np.int32)])
        ov = np.concatenate([ov, np.zeros(len(extra))])
    go = np.zeros((len(cls), C), np.float32)
    go[np.arange(len(cls)), np.maximum(cls, 0) % C] = ov
    return {'boxes': gt.astype(dtype), 'gt_classes': cls, 'gt_overlaps': go}


def bound_boxes(bound, k, seed):
    """k float32 boxes whose float32 area is exactly `bound` while the float64 area of the same corners is not."""
    rng = np.random.RandomState(seed)
    out = []
    s = np.sqrt(bound)
    while len(out) < k:
        x1, y1 = rng.uniform(0, 50, 2).astype(np.float32)
        w = np.float32(s * rng.uniform(0.5, 2.0))
        h = np.float32(bound / float(w))
        b = np.array([x1, y1, x1 + w - 1, y1 + h - 1], np.float32)
        a32 = (b[2] - b[0] + 1) * (b[3] - b[1] + 1)
        a64 = (np.float64(b[2]) - b[0] + 1) * (np.float64(b[3]) - b[1] + 1)
        if a32 == np.float32(bound) and a64 != bound:
            out.append(b)
    return np.array(out, np.float32)


def case_hand():
    """Hand-made: every tie and boundary rule in a few images; uint16 GTs, float32 candidate boxes."""
    r, cand = [], []
    # 0: duplicate GTs and duplicate proposals, several columns at the same maximum; an IoU of exactly 0.5 and 0.6
    r.append(entry([[0, 0, 9, 9], [0, 0, 9, 9], [20, 20, 29, 29], [40, 40, 49, 49]], [1, 1, 2, 3]))
    cand.append([[0, 0, 9, 4], [0, 0, 9, 4], [20, 20, 29, 25], [20, 20, 29, 25], [40, 40, 49, 49], [0, 0, 9, 9]])
    # 1: fewer proposals than GTs, and a round whose best overlap is 0
    r.append(entry([[0, 0, 19, 19], [100, 100, 129, 129], [200, 200, 260, 260]], [1, 2, 1]))
    cand.append([[0, 0, 19, 19], [400, 400, 410, 410]])
    # 2: no proposals (its GTs still count)
    r.append(entry([[10, 10, 59, 59], [0, 0, 4, 4]], [4, 4]))
    cand.append(np.zeros((0, 4), np.float32))
    # 3: no GTs
    r.append(entry(np.zeros((0, 4)), []))
    cand.append([[0, 0, 30, 30], [5, 5, 80, 90]])
    # 4: rows with max(gt_overlaps) < 1 (crowd-style: -1, and 0.5) are not GTs
    r.append(entry([[0, 0, 29, 29], [0, 0, 29, 29], [50, 50, 89, 99]], [1, 2, 3], ovmax=[-1.0, 0.5, 1.0]))
    cand.append([[0, 0, 29, 29], [50, 50, 89, 99], [51, 50, 90, 99]])
    # 5: uint16 GTs over 65535 in area: 300 x 300 -> 24464 (100-200), 256 x 256 -> 0, 400 x 200 -> 14464
    r.append(entry([[0, 0, 299, 299], [10, 10, 265, 265], [0, 0, 399, 199], [0, 0, 199, 199]], [1, 2, 3, 1]))
    cand.append([[0, 0, 299, 299], [10, 10, 265, 260], [0, 0, 399, 199], [5, 5, 199, 199]])
    # 6: float32 proposal areas that round onto 625, 2500 and 10000
    r.append(entry([[0, 0, 24, 24], [0, 0, 49, 49], [0, 0, 99, 99]], [1, 1, 1]))
    cand.append(np.vstack([bound_boxes(b, 2, 7 + k) for k, b in enumerate((625, 2500, 10000))]))
    # 7: a GT on every range bound (uint16 areas 625, 2500, 10000, 40000) and one just below each
    r.append(entry([[0, 0, 24, 24], [0, 0, 23, 25], [0, 0, 49, 49], [0, 0, 48, 50], [0, 0, 99, 99], [0, 0, 98, 100],
                    [0, 0, 199, 199]], [1, 1, 2, 2, 3, 3, 4]))
    cand.append([[0, 0, 24, 24], [0, 0, 49, 49], [0, 0, 99, 99], [0, 0, 199, 199], [0, 0, 98, 100]])
    cand = [np.asarray(c, np.float32).reshape(-1, 4) for c in cand]
    return r, cand, None, None


def seeded_roidb(seed, n_img, n_prop, n_gt, quant):
    rng = np.random.RandomState(seed)
    r, cand = [], []
    for i in range(n_img):
        W, H = rng.randint(300, 700), rng.randint(300, 700)
        k = rng.poisson(n_gt)
        w = np.exp(rng.uniform(np.log(4), np.log(400), k)).clip(2, W - 2)
        h = (w * np.exp(rng.uniform(-0.7, 0.7, k))).clip(2, H - 2)
        x = rng.uniform(0, W - w)
        y = rng.uniform(0, H - h)
        g = np.round(np.stack([x, y, x + w, y + h], 1))
        if k > 1 and rng.rand() < 0.3:
            g[1] = g[0]  # a duplicate GT
        cls = rng.randint(1, C, k)
        ovm = np.where(rng.rand(k) < 0.1, -1.0, 1.0)
        r.append(entry(g, cls, ovmax=ovm))
        m = rng.randint(0, n_prop) if rng.rand() > 0.05 else 0
        p = np.zeros((m, 4))
        if k and m:
            src = g[rng.randint(k, size=m)]
            p = src + rng.randn(m, 4) * rng.choice([0.5, 4.0, 20.0], size=(m, 1))
        near = rng.rand(m) < 0.3
        p[near | (k == 0)] = np.stack([rng.uniform(0, W - 40, m), rng.uniform(0, H - 40, m),
                                       np.zeros(m), np.zeros(m)], 1)[near | (k == 0)]
        p[:, 2:] = np.maximum(p[:, 2:], p[:, :2] + rng.uniform(1, 120, (m, 2)))
        p = np.round(p * quant) / quant
        if m > 3:
            p[rng.randint(m, size=m // 4)] = p[rng.randint(m, size=m // 4)]  # duplicate proposals
        cand.append(p.astype(np.float32))
    return r, cand


def case_seeded():
    r, cand = seeded_roidb(11, 60, 120, 6, 1)
    return r, cand, None, None


def case_thresholds(T):
    r, cand = seeded_roidb(12, 25, 80, 5, 2)
    rng = np.random.RandomState(100 + T)
    thr = np.sort(rng.uniform(0, 1, T)) if T != 8 else np.array([0.0, 0.1, 0.3, 0.5, 0.5, 0.7, 0.9, 1.0])
    if T == 130:
        thr[:5] = [-0.5, 0.0, 0.5, 0.6000000000000001, 1.0]
    return r, cand, thr, None


def case_merged():
    """candidate_boxes=None on a merged RPN roidb: float32 boxes, GT rows then proposal rows; num_images < len."""
    r, cand = seeded_roidb(13, 30, 60, 4, 4)
    out = []
    for e, p in zip(r, cand):
        boxes = np.vstack([e['boxes'].astype(np.float32), p])
        out.append({'boxes': boxes, 'gt_classes': np.concatenate([e['gt_classes'], np.zeros(len(p), np.int32)]),
                    'gt_overlaps': np.vstack([e['gt_overlaps'], np.zeros((len(p), C), np.float32)])})
    return out, None, None, 27


def case_u16_props():
    """candidate_boxes=None on a uint16 roidb whose proposal rows (class 0) wrap their areas."""
    rng = np.random.RandomState(14)
    r = []
    for i in range(12):
        g = np.array([[0, 0, 299, 299], [20, 30, 140, 200], [5, 5, 260, 270]])[:rng.randint(0, 4)]
        p = np.vstack([g + rng.randint(-10, 10, g.shape), [[0, 0, 255, 255], [0, 0, 24, 24], [3, 3, 330, 330]]])
        p = np.clip(p, 0, 600)
        p[:, 2:] = np.maximum(p[:, 2:], p[:, :2])
        r.append(entry(g, rng.randint(1, C, len(g)), extra=p))
    return r, None, None, None


CASES = {
    "hand": case_hand,
    "seeded": case_seeded,
    "thr1": lambda: case_thresholds(1),
    "thr8": lambda: case_thresholds(8),
    "thr9": lambda: case_thresholds(9),
    "thr130": lambda: case_thresholds(130),
    "merged": case_merged,
    "u16props": case_u16_props,
}


class _Imdb(object):
    pass


def run_case(IMDB, rnp, name, out):
    roidb, cand, thr, n_img = CASES[name]()
    imdb = IMDB('synthetic', 'recall', '/nonexistent', '/nonexistent')
    imdb.num_images = len(roidb) if n_img is None else n_img
    rnp.sorts.clear()
    rnp.recalls.clear()
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        text = imdb.evaluate_recall(roidb, candidate_boxes=cand, thresholds=thr)
    assert len(rnp.sorts) == 7 and len(rnp.recalls) == 7, (len(rnp.sorts), len(rnp.recalls))
    assert buf.getvalue() == ''.join(l + '\n' for l in buf.getvalue().split('\n')[:-1])
    k = name + '_'
    out[k + 'n'] = np.array([len(e['boxes']) for e in roidb], np.int64)
    out[k + 'boxes'] = np.concatenate([e['boxes'] for e in roidb])
    out[k + 'gt_classes'] = np.concatenate([e['gt_classes'] for e in roidb])
    out[k + 'gt_overlaps'] = np.concatenate([e['gt_overlaps'] for e in roidb])
    if cand is not None:
        out[k + 'cand_n'] = np.array([len(c) for c in cand], np.int64)
        out[k + 'cand'] = np.concatenate(cand)
    if thr is not None:
        out[k + 'thresholds'] = np.asarray(thr, np.float64)
    out[k + 'num_images'] = np.array(imdb.num_images, np.int64)
    out[k + 'text'] = np.array(text)
    out[k + 'stdout'] = np.array(buf.getvalue())
    out[k + 'recalls'] = np.stack(rnp.recalls).astype(np.float64)
    out[k + 'ov_n'] = np.array([len(s) for s in rnp.sorts], np.int64)
    out[k + 'ov'] = np.concatenate(rnp.sorts).astype(np.float64)


def main():
    IMDB, rnp = load_reference()
    out = {}
    for name in CASES:
        run_case(IMDB, rnp, name, out)
        print(name, 'GT overlaps per range', list(out[name + '_ov_n']))
    np.savez_compressed(OUT, **out)
    print('wrote', os.path.relpath(OUT), os.path.getsize(OUT), 'bytes')


if __name__ == "__main__":
    sys.exit(main())
