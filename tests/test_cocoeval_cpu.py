"""COCO box evaluation without a device: the numpy restatement (oracle/cocoeval_np.py), the host CSR packing, the
results writer and gt_roidb against the reference's own pycocotools / lib/dataset/coco.py (tests/golden/cocoeval_ref.npz,
oracle/run_ref_cocoeval.py), and the argument checks of the three entry points of csrc/coco_eval.cu.

The argument tests pass fabricated, never dereferenced device addresses (as test_rowkernel_args_cpu.py does): every call
violates one rule and must return from the check before any CUDA call; an empty input must return 0 without a launch."""
import ctypes
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", "oracle"))

import cocoeval_fixture as F  # noqa: E402
import cocoeval_np  # noqa: E402
from sniper_b200 import _lib, cocoeval  # noqa: E402
from sniper_b200 import coco as coco_imdb  # noqa: E402


@pytest.fixture(scope="module")
def fx():
    return F.load()


def _restated(fx, name):
    cg, cd, p = F.cocos(fx, name)
    p.imgIds, p.catIds = sorted(cg.getImgIds()), sorted(cg.getCatIds())
    pk = cocoeval.pack(cg, cd, p)
    r = cocoeval_np.match(pk, p.iouThrs, p.areaRng)
    return pk, r, p


@pytest.mark.parametrize("name", F.CASES)
def test_restatement_equals_reference(fx, name):
    pk, r, p = _restated(fx, name)
    F.assert_evalimgs_equal(F.flat_evalimgs(F.evalimgs_from_match(pk, r, p)), fx, name)
    prec, rec = cocoeval_np.accumulate(pk, r, p.maxDets, p.recThrs, pk['K'])
    assert prec.tobytes() == fx[name + "_precision"].tobytes()
    assert rec.tobytes() == fx[name + "_recall"].tobytes()
    if name + "_stats" in fx:
        E = cocoeval.COCOeval()
        E.params = p
        E.eval = dict(precision=prec, recall=rec)
        assert np.asarray(E.summarize()).tobytes() == fx[name + "_stats"].tobytes()


def test_restatement_iou_equals_bbiou(fx):
    for name in ("hand", "synth"):
        pk, _, p = _restated(fx, name)
        keys = {(int(i), int(c)) for i, c in fx[name + "_iou_keys"]}
        off = np.concatenate([[0], np.cumsum(np.prod(fx[name + "_iou_shape"], 1))])
        got = {}
        for q in range(pk['P']):
            d0, d1, g0, g1 = pk['dt_off'][q], pk['dt_off'][q + 1], pk['gt_off'][q], pk['gt_off'][q + 1]
            if d1 > d0 and g1 > g0:
                key = (int(p.imgIds[pk['pair_img'][q]]), int(p.catIds[pk['pair_cat'][q]]))
                got[key] = cocoeval_np.bb_iou(pk['dt_box'][d0:d1, None], pk['gt_box'][None, g0:g1],
                                              (pk['gt_flags'][g0:g1] & 1) != 0)
        assert set(got) == keys
        for j, (i, c) in enumerate(fx[name + "_iou_keys"]):
            assert got[int(i), int(c)].tobytes() == fx[name + "_iou_flat"][off[j]:off[j + 1]].tobytes()


@pytest.mark.parametrize("name", F.CASES)
def test_pack_follows_cocoeval_grouping(fx, name):
    """GT rows of a pair in _gts order; detection rows in evaluateImg's sorted(dt, key=-score)[:maxDet] order."""
    pk, _, p = _restated(fx, name)
    gts = {}
    k0 = 0
    for (i, c), n in zip(fx[name + "_gts_keys"], fx[name + "_gts_n"]):
        if n:  # the reference's defaultdict also holds the empty pairs its lookups created
            gts[int(i), int(c)] = fx[name + "_gts_ids"][k0:k0 + n].tolist()
        k0 += n
    got = {}
    for q in range(pk['P']):
        if pk['gt_off'][q + 1] > pk['gt_off'][q]:
            got[int(p.imgIds[pk['pair_img'][q]]), int(p.catIds[pk['pair_cat'][q]])] = \
                pk['gt_id'][pk['gt_off'][q]:pk['gt_off'][q + 1]].tolist()
    assert got == gts
    # the pairs are category-major, then image order
    assert np.all(np.diff(pk['pairs']) > 0)
    dt = F.flat_evalimgs(F.evalimgs_from_match(pk, cocoeval_np.match(pk, p.iouThrs, p.areaRng), p))
    assert dt['ev_dtIds'].tobytes() == fx[name + "_ev_dtIds"].tobytes()
    assert dt['ev_dtScores'].tobytes() == fx[name + "_ev_dtScores"].tobytes()


def _imdb(tmp_path, gt, image_set="val2017"):
    ann = tmp_path / "data" / "annotations"
    ann.mkdir(parents=True)
    (ann / ("instances_%s.json" % image_set)).write_text(json.dumps(gt))
    imgs = tmp_path / "data" / "images" / image_set
    imgs.mkdir(parents=True)
    for im in gt['images']:
        (imgs / ("COCO_%s_%012d.jpg" % (image_set, im['id']))).write_bytes(b"")
    return coco_imdb.coco(image_set, str(tmp_path), str(tmp_path / "data"), device="cpu")


def _all_boxes(fx, n_img):
    nb = fx["synth_boxes_n"]
    flat, k0 = fx["synth_boxes"], 0
    out = [[None] * n_img for _ in range(nb.shape[0])]
    for k in range(nb.shape[0]):
        for i in range(n_img):
            out[k][i] = flat[k0:k0 + nb[k, i]]
            k0 += nb[k, i]
    return out


def test_writer_rows_equal_reference(fx, tmp_path):
    gt = json.loads(bytes(fx["synth_gt_json"]).decode())
    imdb = _imdb(tmp_path, gt)
    assert imdb.image_set_index == fx["synth_image_set_index"].tolist()
    all_boxes = _all_boxes(fx, imdb.num_images)
    res = str(tmp_path / "res.json")
    imdb._write_coco_results(all_boxes, res)
    rows = json.load(open(res))
    assert [r['image_id'] for r in rows] == fx["synth_rows_image_id"].tolist()
    assert [r['category_id'] for r in rows] == fx["synth_rows_category_id"].tolist()
    assert np.array([r['bbox'] for r in rows]).tobytes() == fx["synth_rows_bbox"].tobytes()
    assert np.array([r['score'] for r in rows]).tobytes() == fx["synth_rows_score"].tobytes()
    assert all(sorted(r) == ['bbox', 'category_id', 'image_id', 'score'] for r in rows)
    # the case holds values on which Python 3's round would differ from the reference's 2.7 round
    d = np.concatenate([b for k in all_boxes[1:] for b in k]).astype(np.float64)
    xywh = np.stack([d[:, 0], d[:, 1], d[:, 2] - d[:, 0] + 1, d[:, 3] - d[:, 1] + 1], 1)
    py3 = np.array([[round(v, 1) for v in r] for r in xywh.tolist()])
    assert (py3 != fx["synth_rows_bbox"]).any()
    assert any(round(s, 8) != r for s, r in zip(d[:, 4].tolist(), fx["synth_rows_score"].tolist()))


def test_round_py2_ties():
    x = np.array([123.25, -123.25, 0.05, 0.15, 0.25, 2.675, 1 / 512.0, 0.5 / 1e8, -0.04, 7.0])
    assert coco_imdb.round_py2(x[:6], 1).tolist() == [123.3, -123.3, 0.1, 0.1, 0.3, 2.7]
    assert coco_imdb.round_py2(x[6:8], 8).tolist() == [0.00195313, 1e-08]
    assert str(coco_imdb.round_py2(x[8:9], 1)[0]) == "-0.0"


def test_gt_roidb_equals_reference(fx, tmp_path):
    gt = json.loads(bytes(fx["synth_gt_json"]).decode())
    imdb = _imdb(tmp_path, gt)
    roidb = imdb.gt_roidb()
    assert [[r['height'], r['width']] for r in roidb] == fx["roidb_hw"].tolist()
    for f in ('boxes', 'boxesc', 'gt_classes', 'gt_overlaps', 'max_classes', 'max_overlaps'):
        got = np.concatenate([r[f] for r in roidb])
        ref = fx["roidb_" + f]
        assert got.dtype == ref.dtype and got.shape == ref.shape and got.tobytes() == ref.tobytes(), f
        assert [len(r[f]) for r in roidb] == fx["roidb_%s_n" % f].tolist()
    assert all(os.path.exists(r['image']) and r['flipped'] is False for r in roidb)
    # the second call reads the cache
    again = imdb.gt_roidb()
    assert all(a['boxes'].tobytes() == b['boxes'].tobytes() for a, b in zip(again, roidb))


def test_refusals_on_host():
    gt, res, _ = F.case(F.load(), "hand")
    cg = cocoeval.COCO(gt)
    with pytest.raises(ValueError, match="empty"):
        cg.loadRes([])
    with pytest.raises(AssertionError):
        cg.loadRes([dict(image_id=999, category_id=1, bbox=[0, 0, 1, 1], score=0.5)])
    for field, msg in (("useSegm", "useSegm"), ("useCats", "useCats")):
        E = cocoeval.COCOeval(cg, cg.loadRes(json.loads(json.dumps(res))))
        setattr(E.params, field, 1 if field == "useSegm" else 0)
        with pytest.raises(NotImplementedError, match=msg):
            E.evaluate()
    assert cocoeval.Params().iouThrs[8] == 0.8999999999999999


# ---------------------------------------------------------------------------------------------------------------------
# argument checks (fabricated device pointers; never dereferenced)
# ---------------------------------------------------------------------------------------------------------------------
A_ = 0x7f0000100000
V = [A_ + 0x10000 * i for i in range(1, 24)]


def _h(a, t):
    a = np.ascontiguousarray(a, dtype=t)
    return a, a.ctypes.data


def _call(name, **kw):
    L = _lib.lib()
    return getattr(L, name)(*kw.values()), L.sniper_last_error().decode()


def _iou_args(**over):
    dt_off, dp = _h([0, 2, 3], np.int32)
    gt_off, gp = _h([0, 1, 3], np.int32)
    iou_off, ip = _h([0, 2, 4], np.int64)      # pair 0: 2 x 1, pair 1: 1 x 2
    kw = dict(dt_box=V[0], gt_box=V[1], gt_flags=V[2], dt_off=V[3], gt_off=V[4], iou_off=V[5], dt_off_host=dp,
              gt_off_host=gp, iou_off_host=ip, P=2, out=V[6], stream=0)
    kw.update(over)
    return kw, (dt_off, gt_off, iou_off)


def _match_args(**over):
    dt_off, dp = _h([0, 2, 3], np.int32)
    gt_off, gp = _h([0, 1, 3], np.int32)
    thr, tp = _h([0.5, 0.75], np.float64)
    rng, rp = _h([0, 1e10, 0, 1024], np.float64)
    kw = dict(dt_box=V[0], dt_area=V[1], dt_id=V[2], gt_box=V[3], gt_area=V[4], gt_flags=V[5], gt_id=V[6],
              dt_off=V[7], gt_off=V[8], dt_off_host=dp, gt_off_host=gp, P=2, iou_thrs=tp, T=2, area_rng=rp, A=2,
              dt_flags=V[9], npig=V[10], gt_match=V[11], dt_match=0, gt_order=0, stream=0)
    kw.update(over)
    return kw, (dt_off, gt_off, thr, rng)


def _acc_args(**over):
    dt_off, dp = _h([0, 2, 3], np.int32)
    cpo, cp = _h([0, 1, 2], np.int32)
    md, mp = _h([1, 10, 100], np.int32)
    rt, rp = _h(np.linspace(0, 1, 101), np.float64)
    kw = dict(dt_flags=V[0], dt_rank=V[1], cat_order=V[2], dt_off=V[3], npig=V[4], cat_pair_off=V[5],
              dt_off_host=dp, cat_pair_off_host=cp, K=2, P=2, A=4, T=10, max_dets=mp, M=3, rec_thrs=rp, R=101,
              precision=V[6], recall=V[7], stream=0)
    kw.update(over)
    return kw, (dt_off, cpo, md, rt)


def _bad(kwkeep, name, pattern):
    kw, keep = kwkeep
    rc, msg = _call(name, **kw)
    assert rc == -1, (name, kw)
    assert pattern in msg, (pattern, msg)


def test_iou_refusals():
    n = "sniper_coco_box_iou_batched"
    _bad(_iou_args(P=-1), n, "P (-1) must not be negative")
    _bad(_iou_args(dt_off_host=0), n, "host offsets")
    bad, bp = _h([0, 3, 2], np.int32)
    _bad(_iou_args(dt_off_host=bp), n, "dt_off must start at 0 and not decrease")
    bad2, bp2 = _h([1, 2, 3], np.int32)
    _bad(_iou_args(gt_off_host=bp2), n, "gt_off must start at 0")
    wrong, wp = _h([0, 2, 3], np.int64)
    _bad(_iou_args(iou_off_host=wp), n, "iou_off of pair 1")
    _bad(_iou_args(iou_off=0), n, "dt_off / gt_off / iou_off must not be null")
    _bad(_iou_args(gt_flags=0), n, "dt_box / gt_box / gt_flags must not be null")
    _bad(_iou_args(out=0), n, "out must not be null")
    assert _call(n, **_iou_args(P=0)[0])[0] == 0


def test_match_refusals():
    n = "sniper_coco_match"
    _bad(_match_args(P=-2), n, "P (-2) must not be negative")
    _bad(_match_args(T=0), n, "T (0 IoU thresholds)")
    _bad(_match_args(T=65), n, "T (65 IoU thresholds)")
    _bad(_match_args(A=0), n, "A (0 area ranges)")
    _bad(_match_args(iou_thrs=0), n, "iou_thrs / area_rng (host) must not be null")
    _bad(_match_args(gt_off_host=0), n, "host offsets")
    bad, bp = _h([0, 2, 1], np.int32)
    _bad(_match_args(dt_off_host=bp), n, "dt_off must start at 0 and not decrease")
    _bad(_match_args(gt_off_host=bp), n, "gt_off must start at 0 and not decrease")
    _bad(_match_args(npig=0), n, "dt_off / gt_off / npig must not be null")
    _bad(_match_args(dt_area=0), n, "dt_box / dt_area / dt_id / dt_flags must not be null")
    _bad(_match_args(gt_match=0), n, "gt_box / gt_area / gt_flags / gt_id / gt_match must not be null")
    assert _call(n, **_match_args(P=0)[0])[0] == 0


def test_accumulate_refusals():
    n = "sniper_coco_accumulate"
    _bad(_acc_args(K=-1), n, "must not be negative")
    _bad(_acc_args(T=0), n, "T (0 IoU thresholds)")
    _bad(_acc_args(M=0), n, "M (0 maxDets)")
    _bad(_acc_args(R=0), n, "R (0 recall thresholds)")
    _bad(_acc_args(A=17), n, "A (17 area ranges)")
    md, mp = _h([1, 100, 10], np.int32)
    _bad(_acc_args(max_dets=mp), n, "maxDets must be sorted")
    rt, rp = _h([0, 0.5, 0.25], np.float64)
    _bad(_acc_args(rec_thrs=rp, R=3), n, "recThrs must be sorted")
    _bad(_acc_args(rec_thrs=0), n, "max_dets / rec_thrs (host) must not be null")
    cpo, cp = _h([0, 2, 1], np.int32)
    _bad(_acc_args(cat_pair_off_host=cp), n, "cat_pair_off must start at 0, not decrease and end at P")
    cpo2, cp2 = _h([0, 1, 1], np.int32)
    _bad(_acc_args(cat_pair_off_host=cp2), n, "end at P (2)")
    bad, bp = _h([0, 2, 1], np.int32)
    _bad(_acc_args(dt_off_host=bp), n, "dt_off must start at 0 and not decrease")
    _bad(_acc_args(npig=0), n, "cat_pair_off / dt_off / npig must not be null")
    _bad(_acc_args(cat_order=0), n, "dt_flags / dt_rank / cat_order must not be null")
    _bad(_acc_args(recall=0), n, "precision / recall must not be null")
    assert _call(n, **_acc_args(K=0)[0])[0] == 0
