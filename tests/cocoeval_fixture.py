"""Shared helpers of the COCO evaluation tests: the cases of tests/golden/cocoeval_ref.npz (written by
oracle/run_ref_cocoeval.py from the reference's own pycocotools) and the flat form its evalImgs are stored in."""
import json
import os

import numpy as np

from sniper_b200 import cocoeval

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cocoeval_ref.npz")
CASES = ("hand", "synth", "params")


def load():
    return dict(np.load(GOLDEN))


def case(fx, name):
    """(gt dataset dict, results list, Params) of a fixture case: synth and params share the synth set and its
    results rows."""
    src = "synth" if name == "params" else name
    gt = json.loads(bytes(fx[src + "_gt_json"]).decode())
    if src == "hand":
        res = json.loads(bytes(fx["hand_res_json"]).decode())
    else:
        res = [dict(image_id=int(i), category_id=int(c), bbox=b.tolist(), score=float(s))
               for i, c, b, s in zip(fx["synth_rows_image_id"], fx["synth_rows_category_id"], fx["synth_rows_bbox"],
                                     fx["synth_rows_score"])]
    p = cocoeval.Params()
    p.iouThrs = fx[name + "_iouThrs"]
    p.recThrs = fx[name + "_recThrs"]
    p.maxDets = fx[name + "_maxDets"].tolist()
    p.areaRng = fx[name + "_areaRng"].tolist()
    return gt, res, p


def cocos(fx, name):
    gt, res, p = case(fx, name)
    cg = cocoeval.COCO(gt)
    cd = cg.loadRes(res)
    return cg, cd, p


def flat_evalimgs(E):
    """evalImgs -> the fixture's ev_* arrays (entries that are not None, concatenated)."""
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


def evalimgs_from_match(pk, r, p):
    """cocoeval's evalImgs list rebuilt from match outputs (dt_flags, dt_match, gt_match, gt_order) on pack's CSR."""
    I, A = pk['I'], len(p.areaRng)
    out = [None] * (pk['K'] * A * I)
    for q in range(pk['P']):
        g0, g1, d0, d1 = pk['gt_off'][q], pk['gt_off'][q + 1], pk['dt_off'][q], pk['dt_off'][q + 1]
        for a in range(A):
            order = r['gt_order'][a, g0:g1]
            lo, hi = p.areaRng[a]
            ar = pk['gt_area'][g0:g1][order]
            out[(pk['pair_cat'][q] * A + a) * I + pk['pair_img'][q]] = dict(
                dtIds=pk['dt_id'][d0:d1].tolist(), gtIds=pk['gt_id'][g0:g1][order].tolist(),
                dtScores=pk['dt_score'][d0:d1].tolist(),
                dtMatches=r['dt_match'][a, :, d0:d1].astype(np.float64),
                gtMatches=r['gt_match'][a, :, g0:g1].astype(np.float64),
                gtIgnore=((pk['gt_flags'][g0:g1][order] & 3 != 0) | (ar < lo) | (ar > hi)).astype(np.int64),
                dtIgnore=(r['dt_flags'][a, :, d0:d1] & 2) != 0)
    return out


def assert_evalimgs_equal(flat, fx, name):
    for k, v in flat.items():
        ref = fx[name + "_" + k]
        assert v.shape == ref.shape, (name, k, v.shape, ref.shape)
        assert v.tobytes() == ref.astype(v.dtype).tobytes(), (name, k)


def synthetic_set(seed, n_img=5000, n_cat=80, gt_per_img=7.0, dt_per_img=100):
    """A seeded val2017-shaped set: n_img images, n_cat categories with COCO's id gaps, ~gt_per_img GTs per image (some
    crowd, some `ignore`, areas at the 32^2 / 96^2 edges), dt_per_img detections per image (half near a GT, scores on a
    1/1024 grid for ties).  Returns (gt dataset dict, results list)."""
    rs = np.random.RandomState(seed)
    cat_ids = [c for c in range(1, 91) if c not in (12, 26, 29, 30, 45, 66, 68, 69, 71, 83)][:n_cat]
    imgs = [dict(id=int(i), width=640, height=480) for i in rs.choice(600000, n_img, replace=False)]
    n_gt = rs.poisson(gt_per_img, n_img)
    G = int(n_gt.sum())
    g_img = np.repeat([im['id'] for im in imgs], n_gt)
    g_cat = rs.choice(cat_ids, G, p=np.r_[0.25, np.full(len(cat_ids) - 1, 0.75 / (len(cat_ids) - 1))])
    wh = np.exp(rs.uniform(1.5, 5.5, (G, 2))).round(1)
    wh[rs.rand(G) < 0.02] = [32, 32]
    wh[rs.rand(G) < 0.02] = [96, 96]
    xy = rs.uniform(0, 400, (G, 2)).round(2)
    area = wh[:, 0] * wh[:, 1]
    odd = rs.rand(G) < 0.1
    area[odd] *= rs.uniform(0.5, 1.0, odd.sum())
    crowd = (rs.rand(G) < 0.01).astype(int)
    ign = rs.rand(G) < 0.01
    anns = [dict(id=int(i + 1), image_id=int(g_img[i]), category_id=int(g_cat[i]),
                 bbox=[float(xy[i, 0]), float(xy[i, 1]), float(wh[i, 0]), float(wh[i, 1])], area=float(area[i]),
                 iscrowd=int(crowd[i]), **({'ignore': 1} if ign[i] else {})) for i in range(G)]
    D = n_img * dt_per_img
    d_img = np.repeat([im['id'] for im in imgs], dt_per_img)
    near = rs.rand(D) < 0.5
    src = rs.randint(0, max(G, 1), D)
    dbox = np.concatenate([rs.uniform(0, 400, (D, 2)), np.exp(rs.uniform(1.5, 5.5, (D, 2)))], 1)
    if G:
        jit = dbox.copy()
        jit[:, :2] = xy[src] + rs.normal(0, 3, (D, 2))
        jit[:, 2:] = wh[src] * rs.uniform(0.8, 1.2, (D, 2))
        dbox = np.where(near[:, None], jit, dbox)
        d_img = np.where(near, g_img[src], d_img)
    d_cat = np.where(near & (rs.rand(D) < 0.8), g_cat[src] if G else 1, rs.choice(cat_ids, D))
    score = rs.randint(0, 1024, D) / 1024.0
    dbox = dbox.round(1)
    res = [dict(image_id=int(d_img[i]), category_id=int(d_cat[i]), bbox=dbox[i].tolist(), score=float(score[i]))
           for i in range(D)]
    cats = [dict(id=int(c), name="c%d" % c, supercategory="s") for c in cat_ids]
    return dict(images=imgs, categories=cats, annotations=anns), res
