"""TEST INFRASTRUCTURE ONLY.  Runs the reference's OWN COCO evaluation in THIS container and writes
tests/golden/cocoeval_ref.npz (run: python oracle/run_ref_cocoeval.py):

  COCO, loadRes                            lib/dataset/pycocotools/coco.py
  COCOeval, Params                         lib/dataset/pycocotools/cocoeval.py, with mask.iou -> bbIou of
                                           lib/dataset/pycocotools/maskApi.c compiled as it lies into
                                           oracle/_ref/libref_maskapi.so and called through ctypes (what _mask.pyx
                                           does for box inputs: float64 arrays, bbIou, reshape (m, n) in Fortran order)
  coco_results_one_category_kernel,        lib/dataset/coco.py:21-59, 153-260
  coco._load_coco_annotation

_mask.pyx itself is not used: its `iou` marks a malloc'ed buffer NPY_OWNDATA, which numpy 2's allocator does not own
(the process aborts with a double free at exit).  The sources are read as text from /root/reference and executed in
memory (nothing is copied into the repo); Python-2-only tokens are rewritten (print statements, tuple-parameter
lambdas, xrange, np.float, filter(), the float sample count of np.linspace).  `round` is bound to Python 2.7's: the
exact binary value rounded half away from zero (decimal ROUND_HALF_UP on Decimal(float)), which is what the reference
ran under; Python 3's round differs on exact ties.  The arithmetic and the control flow are the reference's."""
import ctypes
import json
import os
import re
import subprocess
import sys
import tempfile
import textwrap
import types
from decimal import ROUND_HALF_UP, Decimal

import numpy as np

REF = "/root/reference"
PCT = os.path.join(REF, "lib", "dataset", "pycocotools")
HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_ref", "libref_maskapi.so")
OUT = os.path.join(HERE, "..", "tests", "golden", "cocoeval_ref.npz")


def py2_round(x, n=0):
    return float(Decimal(float(x)).quantize(Decimal(1).scaleb(-n), rounding=ROUND_HALF_UP))


def _py3(src):
    src = re.sub(r'^(\s*)print (.+)$', r'\1print(\2)', src, flags=re.M)
    src = re.sub(r'\bnp\.float\b', 'np.float64', src)
    src = src.replace('xrange(', 'range(')
    src = src.replace('lambda (ind, g): g[\'_ignore\']', 'lambda ig: ig[1][\'_ignore\']')
    src = src.replace('E = filter(None, E)', 'E = list(filter(None, E))')
    src = src.replace('np.round((0.95-.5)/.05)+1', 'int(np.round((0.95-.5)/.05)+1)')
    src = src.replace('np.round((1.00-.0)/.01)+1', 'int(np.round((1.00-.0)/.01)+1)')
    return src


def _maskapi():
    if not os.path.exists(LIB):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-std=c99", "-ffp-contract=off", "-o", LIB,
                               os.path.join(PCT, "maskApi.c"), "-lm"])
    L = ctypes.CDLL(LIB)
    L.bbIou.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_ulong, ctypes.c_ulong, ctypes.c_void_p,
                        ctypes.c_void_p]
    L.bbIou.restype = None

    def iou(dt, gt, iscrowd):
        if len(dt) == 0 or len(gt) == 0:
            return []
        d = np.ascontiguousarray(np.array(dt, dtype=np.double).reshape(-1, 4))
        g = np.ascontiguousarray(np.array(gt, dtype=np.double).reshape(-1, 4))
        c = np.ascontiguousarray(np.array(iscrowd, dtype=np.uint8))
        o = np.zeros(d.shape[0] * g.shape[0])
        L.bbIou(d.ctypes.data, g.ctypes.data, d.shape[0], g.shape[0], c.ctypes.data, o.ctypes.data)
        return o.reshape((d.shape[0], g.shape[0]), order='F')
    mod = types.ModuleType("mask")
    mod.iou = iou
    return mod


def load_reference():
    """(COCO, COCOeval, coco_results_one_category_kernel, _load_coco_annotation) of the reference."""
    mask = _maskapi()
    ns_coco = {"__name__": "ref_coco"}
    src = open(os.path.join(PCT, "coco.py")).read()
    src = re.sub(r'^(import matplotlib|from matplotlib|from skimage|import urllib|import mask).*$', '', src, flags=re.M)
    ns_coco["mask"] = mask
    exec(compile(_py3(src), "ref/coco.py", "exec"), ns_coco)
    ns_eval = {"__name__": "ref_cocoeval", "mask": mask}
    src = re.sub(r'^import mask$', '', open(os.path.join(PCT, "cocoeval.py")).read(), flags=re.M)
    exec(compile(_py3(src), "ref/cocoeval.py", "exec"), ns_eval)
    ds = open(os.path.join(REF, "lib", "dataset", "coco.py")).read()
    a = ds.index("def coco_results_one_category_kernel")
    b = ds.index("class coco(IMDB)")
    c = ds.index("    def _load_coco_annotation")
    e = ds.index("    def evaluate_detections")
    ns = {"np": np, "round": py2_round}
    exec(compile(_py3(ds[a:b]) + "\n" + _py3(textwrap.dedent(ds[c:e])), "ref/dataset_coco.py", "exec"), ns)
    return ns_coco["COCO"], ns_eval["COCOeval"], ns["coco_results_one_category_kernel"], ns["_load_coco_annotation"]


# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------
def _ann(i, img, cat, box, area=None, crowd=0, **kw):
    a = dict(id=i, image_id=img, category_id=cat, bbox=[float(v) for v in box],
             area=float(box[2] * box[3] if area is None else area), iscrowd=crowd, segmentation=[[0, 0, 1, 1, 2, 2]])
    a.update(kw)
    return a


def _res(img, cat, box, score):
    return dict(image_id=img, category_id=cat, bbox=[float(v) for v in box], score=float(score))


def hand_case():
    """Hand-made edge cases, results given directly."""
    cats = [dict(id=c, name="c%d" % c, supercategory="s") for c in (1, 3, 7, 8)]
    imgs = [dict(id=i, width=640, height=480, file_name="%d.jpg" % i) for i in (10, 11, 12, 13, 14)]
    anns = [
        _ann(0, 10, 1, [0, 0, 10, 10]),                     # annotation id 0: a match to it counts as unmatched
        _ann(5, 10, 1, [0, 0, 10, 10]),                     # same box: equal IoU, the later GT wins
        _ann(6, 10, 1, [100, 100, 20, 10]),                 # a det at IoU exactly 0.5
        _ann(7, 11, 1, [0, 0, 12, 4]),                      # a det at IoU exactly 0.75
        _ann(8, 11, 3, [50, 50, 40, 40], ignore=1),         # `ignore` field
        _ann(9, 11, 3, [5, 5, 32, 32]),                     # area exactly 32^2
        _ann(10, 11, 3, [200, 200, 96, 96]),                # area exactly 96^2
        _ann(11, 11, 3, [300, 50, 50, 50], area=500.0),     # area field unlike the box
        _ann(12, 12, 3, [0, 0, 100, 100], crowd=1),         # crowd matched by several dets
        _ann(13, 12, 3, [400, 300, 60, 40]),
        _ann(14, 14, 3, [10, 10, 30, 30]),                  # GT, no detections in the image
        _ann(15, 10, 8, [20, 20, 80, 80], crowd=1),         # category 8: crowd GT only
        _ann(16, 12, 1, [30, 30, 40, 40]),
        _ann(17, 12, 1, [32, 30, 40, 40]),
    ]
    res = [
        _res(10, 1, [0, 0, 10, 10], 0.9), _res(10, 1, [0, 0, 10, 10], 0.9), _res(10, 1, [100, 100, 40, 10], 0.8),
        _res(10, 1, [0, 0, 10, 10], 0.9),
        _res(11, 1, [0, 0, 9, 4], 0.7), _res(11, 1, [0, 0, 12, 4], 0.7),
        _res(11, 3, [50, 50, 40, 40], 0.95), _res(11, 3, [5, 5, 32, 32], 0.6), _res(11, 3, [200, 200, 96, 96], 0.6),
        _res(11, 3, [300, 50, 50, 50], 0.5), _res(11, 3, [0, 0, 8, 8], 0.4), _res(11, 3, [500, 400, 100, 70], 0.3),
        _res(12, 3, [0, 0, 50, 50], 0.9), _res(12, 3, [50, 50, 50, 50], 0.9), _res(12, 3, [10, 10, 20, 20], 0.85),
        _res(12, 3, [400, 300, 60, 40], 0.2), _res(12, 3, [0, 0, 100, 100], 0.2),
        _res(12, 1, [10, 10, -5, 8], 0.6), _res(12, 1, [30, 30, 40, 40], 0.6), _res(12, 1, [31, 30, 40, 40], 0.6),
        _res(13, 1, [5, 5, 20, 20], 0.9), _res(13, 3, [5, 5, 20, 20], 0.9),    # detections, no GT
        _res(10, 7, [0, 0, 10, 10], 0.5), _res(12, 7, [1, 1, 10, 10], 0.5),    # category 7: no GT
        _res(10, 8, [20, 20, 40, 40], 0.8), _res(10, 8, [60, 60, 40, 40], 0.7),
        _res(11, 3, [5, 5, 32, 32], -0.0), _res(11, 3, [5, 5, 31, 32], 0.0),
    ]
    return dict(images=imgs, categories=cats, annotations=anns), res


def synth_case(seed=3):
    """A seeded COCO-shaped set and the detector output all_boxes[class][image] (float32 x1, y1, x2, y2, score) that
    the results writer turns into the results list: coordinates on quarter pixels and scores on multiples of 1/512
    (rounding ties), score ties within and across images, > 100 detections in one (image, category) and > 100 in one
    image across categories, degenerate boxes (x2 < x1)."""
    rs = np.random.RandomState(seed)
    cat_ids = [1, 2, 4, 5, 9, 11]
    cats = [dict(id=c, name="cls%d" % c, supercategory="s") for c in cat_ids]
    img_ids = [3, 8, 21, 22, 40, 41, 57, 60, 77, 90, 91, 105]
    imgs = [dict(id=i, width=int(rs.randint(300, 641)), height=int(rs.randint(200, 481)), file_name="%d.jpg" % i)
            for i in img_ids]
    anns, aid = [], 1
    for im in imgs:
        for _ in range(rs.randint(0, 9)):
            w, h = rs.randint(1, 200, 2).astype(float) + rs.choice([0, .5], 2)
            x, y = rs.randint(0, im['width'] - 20), rs.randint(0, im['height'] - 20)
            crowd = int(rs.rand() < .08)
            area = w * h if rs.rand() < .85 else float(rs.randint(1, 20000))
            a = _ann(aid, im['id'], int(rs.choice(cat_ids[:5])), [x, y, w, h], area=area, crowd=crowd)
            if rs.rand() < .05:
                a['ignore'] = 1
            anns.append(a)
            aid += 1
    anns.append(_ann(aid, imgs[0]['id'], 1, [40, 40, 0, 12]))        # zero width: dropped by gt_roidb
    K = len(cat_ids) + 1
    all_boxes = [[np.zeros((0, 5), np.float32) for _ in imgs] for _ in range(K)]
    by_img = {}
    for a in anns:
        by_img.setdefault(a['image_id'], []).append(a)
    for ii, im in enumerate(imgs):
        gts = by_img.get(im['id'], [])
        for k in range(1, K):
            n = rs.randint(0, 12)
            if ii == 2 and k == 1:
                n = 130
            if ii == 5:
                n = 35
            if n == 0:
                continue
            x1 = rs.randint(0, im['width'] - 10, n) + rs.choice([0, .25, .5, .75], n)
            y1 = rs.randint(0, im['height'] - 10, n) + rs.choice([0, .25, .5, .75], n)
            w = rs.randint(1, 150, n) + rs.choice([0, .25, .75], n)
            h = rs.randint(1, 150, n) + rs.choice([0, .25, .75], n)
            mine = [g for g in gts if g['category_id'] == cat_ids[k - 1]]
            for j in range(min(len(mine), n)):
                gx, gy, gw, gh = mine[j]['bbox']
                x1[j], y1[j] = gx + rs.choice([0, .25, 1, 3]), gy + rs.choice([0, .75, 2])
                w[j], h[j] = gw + rs.choice([-1, 0, .25, 4]), gh + rs.choice([0, 1, -2])
            s = rs.randint(1, 512, n) / 512.0
            s[rs.rand(n) < .3] = rs.choice([0.5, 0.25, 1 / 512.0])
            b = np.stack([x1, y1, x1 + w - 1, y1 + h - 1, s], 1).astype(np.float32)
            if n > 3:
                b[0, 2] = b[0, 0] - 4                      # x2 < x1
            all_boxes[k][ii] = b
    return dict(images=imgs, categories=cats, annotations=anns), all_boxes


# ---------------------------------------------------------------------------------------------------------------------
def _flat_evalimgs(E):
    keep = [i for i, e in enumerate(E) if e is not None]
    es = [E[i] for i in keep]
    T = es[0]['dtMatches'].shape[0] if es else 0
    cat1 = lambda xs: np.concatenate(xs) if xs else np.zeros(0)
    cat2 = lambda xs: np.concatenate([x.reshape(T, -1) for x in xs], 1) if xs else np.zeros((T, 0))
    return dict(
        ev_index=np.array(keep, np.int64), ev_nd=np.array([len(e['dtIds']) for e in es], np.int64),
        ev_ng=np.array([len(e['gtIds']) for e in es], np.int64),
        ev_dtIds=cat1([np.array(e['dtIds'], np.int64) for e in es]).astype(np.int64),
        ev_gtIds=cat1([np.array(e['gtIds'], np.int64) for e in es]).astype(np.int64),
        ev_dtScores=cat1([np.array(e['dtScores'], np.float64) for e in es]).astype(np.float64),
        ev_dtm=cat2([e['dtMatches'] for e in es]).astype(np.float64),
        ev_gtm=cat2([e['gtMatches'] for e in es]).astype(np.float64),
        ev_gtIg=cat1([np.asarray(e['gtIgnore'], np.int64) for e in es]).astype(np.int64),
        ev_dtIg=cat2([np.asarray(e['dtIgnore'], bool) for e in es]).astype(bool))


def run_eval(COCO, COCOeval, gt, res, params=None, summarize=True):
    cg = COCO()
    cg.dataset = json.loads(json.dumps(gt))
    cg.createIndex()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "results.json")
        with open(path, "w") as f:
            json.dump(res, f)
        cd = cg.loadRes(path)
    E = COCOeval(cg, cd)
    E.params.useSegm = 0
    if params:
        for k, v in params.items():
            setattr(E.params, k, v)
    E.evaluate()
    out = dict(iouThrs=np.asarray(E.params.iouThrs), recThrs=np.asarray(E.params.recThrs),
               maxDets=np.array(E.params.maxDets, np.int64), areaRng=np.array(E.params.areaRng, np.float64))
    keys = sorted(k for k, v in E.ious.items() if len(v))
    out['iou_keys'] = np.array(keys, np.int64).reshape(-1, 2)
    out['iou_shape'] = np.array([E.ious[k].shape for k in keys], np.int64).reshape(-1, 2)
    out['iou_flat'] = np.concatenate([E.ious[k].ravel() for k in keys]) if keys else np.zeros(0)
    gkeys = sorted(E._gts.keys())
    out['gts_keys'] = np.array(gkeys, np.int64).reshape(-1, 2)
    out['gts_n'] = np.array([len(E._gts[k]) for k in gkeys], np.int64)
    out['gts_ids'] = np.array([g['id'] for k in gkeys for g in E._gts[k]], np.int64)
    out.update(_flat_evalimgs(E.evalImgs))
    E.accumulate()
    out['precision'], out['recall'] = E.eval['precision'], E.eval['recall']
    if summarize:
        out['stats'] = np.asarray(E.summarize(), np.float64)
    return out


def main():
    COCO, COCOeval, writer, load_ann = load_reference()
    fx = {}
    gt, res = hand_case()
    for k, v in run_eval(COCO, COCOeval, gt, res).items():
        fx['hand_' + k] = v
    fx['hand_gt_json'] = np.frombuffer(json.dumps(gt).encode(), np.uint8)
    fx['hand_res_json'] = np.frombuffer(json.dumps(res).encode(), np.uint8)

    gt, all_boxes = synth_case()
    cg = COCO()
    cg.dataset = json.loads(json.dumps(gt))
    cg.createIndex()
    cat_ids = cg.getCatIds()
    image_set_index = cg.getImgIds()
    info = [dict(index=i, height=cg.imgs[i]['height'], width=cg.imgs[i]['width']) for i in image_set_index]
    rows = []
    for k, c in enumerate(cat_ids):
        rows += writer(dict(cat_id=c, cls_ind=k + 1, cls='cls%d' % c, ann_type='bbox', binary_thresh=None,
                            all_im_info=info, boxes=all_boxes[k + 1]))
    fx['synth_gt_json'] = np.frombuffer(json.dumps(gt).encode(), np.uint8)
    fx['synth_image_set_index'] = np.array(image_set_index, np.int64)
    nb = np.array([[all_boxes[k][i].shape[0] for i in range(len(info))] for k in range(len(all_boxes))], np.int64)
    fx['synth_boxes_n'] = nb
    fx['synth_boxes'] = np.concatenate([all_boxes[k][i] for k in range(len(all_boxes)) for i in range(len(info))])
    fx['synth_rows_image_id'] = np.array([r['image_id'] for r in rows], np.int64)
    fx['synth_rows_category_id'] = np.array([r['category_id'] for r in rows], np.int64)
    fx['synth_rows_bbox'] = np.array([r['bbox'] for r in rows], np.float64)
    fx['synth_rows_score'] = np.array([r['score'] for r in rows], np.float64)
    res = json.loads(json.dumps(rows))
    for k, v in run_eval(COCO, COCOeval, gt, res).items():
        fx['synth_' + k] = v
    params = dict(maxDets=[1, 10, 100, 300], areaRng=[[0 ** 2, 1e5 ** 2], [0 ** 2, 48 ** 2]])
    for k, v in run_eval(COCO, COCOeval, gt, res, params, summarize=False).items():
        fx['params_' + k] = v

    # gt_roidb fields (_load_coco_annotation) of every image, in image_set_index order
    classes = ['__background__'] + [c['name'] for c in cg.loadCats(cat_ids)]
    self = types.SimpleNamespace(coco=cg, num_classes=len(classes), load_mask=False,
                                 _coco_ind_to_class_ind={c: k + 1 for k, c in enumerate(cat_ids)},
                                 image_path_from_index=lambda index: "img%d" % index)
    recs = [load_ann(self, i)[0] for i in image_set_index]
    for f in ('boxes', 'boxesc', 'gt_classes', 'gt_overlaps', 'max_classes', 'max_overlaps'):
        fx['roidb_' + f] = np.concatenate([r[f] for r in recs])
        fx['roidb_%s_n' % f] = np.array([len(r[f]) for r in recs], np.int64)
    fx['roidb_hw'] = np.array([[r['height'], r['width']] for r in recs], np.int64)
    np.savez_compressed(OUT, **fx)
    print("wrote", os.path.normpath(OUT), os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    sys.exit(main())
