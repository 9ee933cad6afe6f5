"""TEST INFRASTRUCTURE ONLY.  Runs the reference's OWN proposal code in THIS container and writes
tests/golden/proposals_ref.npz (run: python oracle/run_ref_proposals.py, after build_ref_cython.py):

  nmsp                                     lib/nms/nms.py:48-80 (the module imports gpu_nms, so the function is cut out)
  create_roidb_from_box_list, merge_roidbs lib/dataset/imdb.py:145-204, 398-419, with the reference's Cython
                                           bbox_overlaps (oracle/_ref/ref_bbox) behind lib/bbox/bbox_transform.py
  Tester.get_proposals / extract_proposals lib/inference.py:76-98, 372-409, on stub module outputs (the host arithmetic)
  MNIteratorTest.reset                     lib/iterators/MNIteratorTest.py:50-66 (the batch order)

The sources are read as text from /root/reference and the functions cut out and executed in memory (nothing is copied
into the repo); Python-2-only tokens are rewritten: np.float -> float, print statements dropped.  The arithmetic and
the control flow are the reference's."""
import os
import re
import sys
import textwrap
import types

import numpy as np

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "tests", "golden", "proposals_ref.npz")
NUM_CLASSES = 21


def _cut(path, header, indent=""):
    """The text of the definition starting at `header` up to the next definition at the same indentation."""
    src = open(os.path.join(REF, path)).read()
    start = src.index(header)
    m = re.compile(r"\n(%s|)(def |class |@)" % indent).search(src, start + len(header))
    body = src[start:m.start() if m else len(src)]
    body = re.sub(r"np\.float\b", "float", body)
    body = "\n".join(l for l in body.split("\n") if not l.strip().startswith("print "))
    return textwrap.dedent(body)


def load_reference():
    sys.path.insert(0, os.path.join(HERE, "_ref"))
    import ref_bbox
    bt = open(os.path.join(REF, "lib", "bbox", "bbox_transform.py")).read()
    bt = bt.replace("from bbox import bbox_overlaps_cython, ignore_overlaps_cython", "")
    bt = re.sub(r"np\.float\b", "float", bt)
    ns_bt = {"bbox_overlaps_cython": ref_bbox.bbox_overlaps_cython, "ignore_overlaps_cython": ref_bbox.ignore_overlaps_cython}
    exec(compile(bt, "bbox_transform.py", "exec"), ns_bt)
    ns = {"np": np, "bbox_overlaps": ns_bt["bbox_overlaps"], "time": __import__("time"), "os": os}
    for path, header, ind in (("lib/nms/nms.py", "def nmsp(", ""),
                              ("lib/dataset/imdb.py", "    def create_roidb_from_box_list(", "    "),
                              ("lib/dataset/imdb.py", "    def merge_roidbs(", "    "),
                              ("lib/inference.py", "    def get_proposals(", "    "),
                              ("lib/inference.py", "    def extract_proposals(", "    "),
                              ("lib/iterators/MNIteratorTest.py", "    def reset(", "    ")):
        exec(compile(_cut(path, header, ind), path, "exec"), ns)
    return ns


# ---------------------------------------------------------------- inputs
def random_image(rng, n, W=1333, H=800):
    """Clustered boxes (real overlaps) with distinct scores."""
    s = np.exp(rng.uniform(np.log(8), np.log(400), n))
    ar = np.exp(rng.uniform(np.log(0.5), np.log(2.0), n))
    w, h = s * np.sqrt(ar), s / np.sqrt(ar)
    k = max(1, n // 10)
    cx = rng.uniform(0, W, k)[rng.randint(0, k, n)] + rng.randn(n) * 10
    cy = rng.uniform(0, H, k)[rng.randint(0, k, n)] + rng.randn(n) * 10
    d = np.stack([np.clip(cx - w / 2, 0, W - 1), np.clip(cy - h / 2, 0, H - 1), np.clip(cx + w / 2, 0, W - 1),
                  np.clip(cy + h / 2, 0, H - 1), np.zeros(n)], 1).astype(np.float32)
    sc = rng.permutation(n).astype(np.float32) / np.float32(max(n, 1)) + np.float32(1e-3)
    d[:, 4] = sc
    assert len(np.unique(d[:, 4])) == n
    return d


def boundary_image(rng):
    """Pairs of integer boxes whose float32 IoU is exactly float32(0.7) (kept) or the next float32 above it (removed),
    the pair's first box scoring higher; distinct scores."""
    rows = []
    for a_w, a_h, b_w in ((10, 1, 7), (100, 10, 70), (20, 35, 14), (50, 14, 35)):
        for dx, dy in ((0, 0), (300, 200), (600, 50)):
            rows.append([dx, dy, dx + a_w - 1, dy + a_h - 1])
            rows.append([dx, dy, dx + b_w - 1, dy + a_h - 1])
    # pairs whose IoU rounds to just above 0.7: inter 7 / union 9.999.. not representable with integers; search
    for a in range(2, 60):
        for b in range(1, a):
            iou = np.float32(b) / (np.float32(a) + np.float32(b) - np.float32(b))
            if iou > np.float32(0.7) and iou < np.float32(0.71):
                rows.append([900, 10 * len(rows), 900 + a - 1, 10 * len(rows)])
                rows.append([900, 10 * (len(rows) - 1), 900 + b - 1, 10 * (len(rows) - 1)])
                break
        if len(rows) > 40:
            break
    d = np.zeros((len(rows), 5), np.float32)
    d[:, :4] = np.array(rows, np.float32)
    d[:, 4] = (np.arange(len(rows))[::-1] + 1).astype(np.float32) / np.float32(64) + rng.uniform(0, 1e-3, len(rows)) \
        .astype(np.float32)
    assert len(np.unique(d[:, 4])) == len(rows)
    return d


def gt_roidb(rng, props):
    """A GT roidb for the images of `props`: a few boxes, one of them equal to a proposal; some images without GT."""
    out = []
    for i, p in enumerate(props):
        ng = 0 if i % 3 == 2 else int(rng.randint(1, 6))
        boxes = random_image(rng, ng)[:, :4] if ng else np.zeros((0, 4), np.float32)
        if ng and len(p):
            boxes[0] = p[len(p) // 2, :4]                         # a proposal that equals a GT box
        cls = rng.randint(1, NUM_CLASSES, ng).astype(np.int32)
        ov = np.zeros((ng, NUM_CLASSES), np.float32)
        ov[np.arange(ng), cls] = 1
        out.append(dict(image="im%d.jpg" % i, width=1333, height=800, boxes=boxes, gt_classes=cls, gt_overlaps=ov,
                        max_classes=cls.copy(), max_overlaps=np.ones(ng, np.float32), flipped=False))
    return out


def main():
    ns = load_reference()
    rng = np.random.RandomState(0)
    res = {}
    # ---- nmsp
    nms_cases = [random_image(rng, n) for n in (0, 1, 2, 57, 300, 900)] + [boundary_image(rng), random_image(rng, 4096)]
    for c, d in enumerate(nms_cases):
        res["nms_dets_%d" % c] = d
        res["nms_keep_%d" % c] = np.array(ns["nmsp"](d.copy()), dtype=np.int64)
    res["nms_n"] = np.array(len(nms_cases))
    # ---- roidb from the NMS-ed proposals, merged into the GT roidb
    props = [random_image(rng, n) for n in (120, 0, 80, 1, 150, 60)]
    props = [p[np.array(ns["nmsp"](p.copy()), dtype=np.int64)] if len(p) else p for p in props]
    gt = gt_roidb(rng, props)
    imdb = types.SimpleNamespace(num_classes=NUM_CLASSES)
    rpn = ns["create_roidb_from_box_list"](imdb, props, [], gt)
    rpn_scores = [r["proposal_scores"].copy() for r in rpn]
    import copy
    merged = ns["merge_roidbs"](copy.deepcopy(gt), rpn)
    res["roidb_n"] = np.array(len(props))
    for i, (p, g, m) in enumerate(zip(props, gt, merged)):
        res["roidb_props_%d" % i] = p
        res["roidb_gt_boxes_%d" % i] = g["boxes"]
        res["roidb_gt_classes_%d" % i] = g["gt_classes"]
        res["roidb_rpn_scores_%d" % i] = rpn_scores[i]
        for k in ("boxes", "gt_classes", "gt_overlaps", "max_classes", "max_overlaps", "proposal_scores"):
            res["roidb_merged_%s_%d" % (k, i)] = np.asarray(m[k])
    # ---- get_proposals / extract_proposals host arithmetic on stub module outputs
    B, R = 3, 40
    rois = np.zeros((B * R, 5), np.float32)
    rois[:, 0] = np.repeat(np.arange(B), R)
    rois[:, 1:] = rng.uniform(0, 2000, (B * R, 4)).astype(np.float32)
    scores = rng.uniform(0, 1, B * R).astype(np.float32)
    im_info = np.array([[1400, 2000, 1.7504], [1400, 1867, 1.4], [1111, 2000, 2.0 / 3.0]], np.float32)
    im_ids = np.array([2, 0, 1])
    Arr = lambda a: types.SimpleNamespace(asnumpy=lambda: a)                                   # noqa: E731
    out = dict(rois=Arr(rois), scores=Arr(scores), im_ids=Arr(im_ids.astype(np.float32)))
    batch = types.SimpleNamespace(data=[Arr(np.zeros(1)), Arr(im_info), Arr(im_ids)])

    class _Iter(object):
        def __iter__(self):
            return iter([batch])

        def get_batch_size(self):
            return B
    test_iter = _Iter()
    tester = types.SimpleNamespace(num_images=3, batch_size=B, test_iter=test_iter, data_names=["data", "im_info", "im_ids"],
                                   rpn_output_names=dict(rois="rois", scores="scores", im_ids="im_ids"),
                                   forward=lambda b: [out], show_info=lambda s: None, cfg=None)
    tester.get_proposals = types.MethodType(ns["get_proposals"], tester)
    all_boxes = ns["extract_proposals"](tester, n_proposals=25)
    res.update(ext_rois=rois, ext_scores=scores, ext_im_info=im_info, ext_im_ids=im_ids)
    for i in range(3):
        res["ext_boxes_%d" % i] = all_boxes[i]
    # ---- MNIteratorTest.reset order
    orders = []
    for c, (n, bs) in enumerate(((7, 2), (5, 4), (9, 3), (4, 4), (1, 2))):
        wh = rng.randint(100, 1000, (n, 2))
        it = types.SimpleNamespace(roidb=[dict(width=int(w), height=int(h)) for w, h in wh], batch_size=bs)
        ns["reset"](it)
        res["iter_wh_%d" % c], res["iter_bs_%d" % c], res["iter_inds_%d" % c] = wh, np.array(bs), np.asarray(it.inds)
        orders.append(c)
    res["iter_n"] = np.array(len(orders))
    np.savez_compressed(OUT, **res)
    print("wrote", OUT, "keeps:", [len(res["nms_keep_%d" % c]) for c in range(len(nms_cases))])


if __name__ == "__main__":
    main()
