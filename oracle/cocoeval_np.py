"""Vectorised float64 numpy restatement of pycocotools' COCOeval.evaluateImg + accumulate
(lib/dataset/pycocotools/cocoeval.py:189-374) on the CSR of sniper_b200.cocoeval.pack.  Test infrastructure: the GPU
tests compare the device against it at sizes the reference fixture cannot hold.

evaluateImg's greedy loop over the ignore-sorted GTs is restated in closed form per detection: the running best with a
`<` test ends on the LAST occurrence of the maximum IoU among the candidates that reach the threshold; the candidates
are the non-ignored, not-yet-matched (or crowd) GTs, and only when none of them reaches the threshold do the ignored
ones compete (the loop breaks at the first ignored GT once a regular match exists).  Detections stay sequential.
"""
import numpy as np


def bb_iou(d, g, crowd):
    """bbIou (maskApi.c:98-109) with broadcasting: d [..., 4], g [..., 4] xywh, crowd bool."""
    ga = g[..., 2] * g[..., 3]
    da = d[..., 2] * d[..., 3]
    w = np.minimum(d[..., 2] + d[..., 0], g[..., 2] + g[..., 0]) - np.maximum(d[..., 0], g[..., 0])
    h = np.minimum(d[..., 3] + d[..., 1], g[..., 3] + g[..., 1]) - np.maximum(d[..., 1], g[..., 1])
    i = w * h
    u = np.where(crowd, da, da + ga - i)
    with np.errstate(divide='ignore', invalid='ignore'):
        o = i / u
    return np.where((w <= 0) | (h <= 0), 0.0, o)


def _last_argmax(v):
    return v.shape[-1] - 1 - np.argmax(v[..., ::-1], axis=-1)


def match(pk, iouThrs, areaRng, chunk=4096):
    """evaluateImg for every pair x area x threshold -> dict(dt_flags [A, T, Dtot] uint8 (bit 0 matched, bit 1
    ignored), npig [P, A], gt_match [A, T, Gtot] (dt ids, ignore-sorted order), dt_match [A, T, Dtot] (gt ids),
    gt_order [A, Gtot])."""
    thr = np.minimum(np.asarray(iouThrs, np.float64), 1 - 1e-10)
    rng = np.asarray(areaRng, np.float64).reshape(-1, 2)
    T, A, P = thr.size, rng.shape[0], pk['P']
    dt_off, gt_off = pk['dt_off'].astype(np.int64), pk['gt_off'].astype(np.int64)
    Dtot, Gtot = int(dt_off[-1]), int(gt_off[-1])
    nd, ng = np.diff(dt_off), np.diff(gt_off)
    out = dict(dt_flags=np.zeros((A, T, Dtot), np.uint8), npig=np.zeros((P, A), np.int32),
               gt_match=np.zeros((A, T, Gtot), np.int64), dt_match=np.zeros((A, T, Dtot), np.int64),
               gt_order=np.zeros((A, Gtot), np.int32))
    crowd_all = (pk['gt_flags'] & 1) != 0
    flag_ig_all = (pk['gt_flags'] & 3) != 0
    by_d = np.argsort(-nd, kind='stable')           # chunks of similar detection counts
    for c0 in range(0, P, chunk):
        ps = by_d[c0:c0 + chunk]
        n = ps.size
        Dm, Gm = int(nd[ps].max()), int(ng[ps].max())
        rows = np.arange(n)
        gl = np.arange(Gm)[None, :]
        gvalid = gl < ng[ps][:, None]
        gidx = np.where(gvalid, gt_off[ps][:, None] + gl, 0)
        dl = np.arange(Dm)[None, :]
        dvalid = dl < nd[ps][:, None]
        didx = np.where(dvalid, dt_off[ps][:, None] + dl, 0)
        ious = bb_iou(pk['dt_box'][didx][:, :, None, :], pk['gt_box'][gidx][:, None, :, :],
                      crowd_all[gidx][:, None, :])                       # [n, Dm, Gm]
        for a in range(A):
            lo, hi = rng[a]
            garea = pk['gt_area'][gidx]
            ig = flag_ig_all[gidx] | (garea < lo) | (garea > hi)
            order = np.argsort(np.where(gvalid, ig.astype(np.int64), 2), axis=1, kind='stable')
            ig_s = np.take_along_axis(ig, order, 1)
            valid_s = np.take_along_axis(gvalid, order, 1)
            crowd_s = np.take_along_axis(crowd_all[gidx], order, 1)
            id_s = np.take_along_axis(pk['gt_id'][gidx], order, 1)
            iou_s = np.take_along_axis(ious, order[:, None, :], 2)
            out['npig'][ps, a] = (valid_s & ~ig_s).sum(1)
            pos = np.nonzero(valid_s)
            out['gt_order'][a, gt_off[ps][pos[0]] + pos[1]] = order[pos]
            gtm = np.zeros((n, T, Gm), np.int64)
            darea = pk['dt_area'][didx]
            for d in range(Dm):
                dv = dvalid[:, d]
                free = valid_s[:, None, :] & ~((gtm > 0) & ~crowd_s[:, None, :])     # [n, T, Gm]
                iou = np.broadcast_to(iou_s[:, d, None, :], free.shape)
                m = np.full((n, T), -1)
                for cand in (free & ~ig_s[:, None, :], free & ig_s[:, None, :]):
                    v = np.where(cand, iou, -np.inf)
                    hit = (m < 0) & (v.max(2, initial=-np.inf) >= thr[None, :]) & dv[:, None]
                    m = np.where(hit, _last_argmax(v), m)
                matched = m >= 0
                mm = np.maximum(m, 0)
                gid = np.where(matched, np.take_along_axis(id_s, mm, 1), 0)
                dig = matched & np.take_along_axis(ig_s, mm, 1)
                r_, t_ = np.nonzero(matched)
                gtm[r_, t_, m[r_, t_]] = pk['dt_id'][didx[r_, d]]
                dig = dig | ((gid == 0) & ((darea[:, d] < lo) | (darea[:, d] > hi))[:, None])
                sel = np.nonzero(dv)[0]
                gd = didx[sel, d]
                out['dt_flags'][a][:, gd] = ((gid[sel] != 0) | (dig[sel].astype(np.uint8) << 1)).T
                out['dt_match'][a][:, gd] = gid[sel].T
            r_, g_ = np.nonzero(valid_s)
            out['gt_match'][a][:, gt_off[ps][r_] + g_] = gtm[r_, :, g_].T
    return out


def accumulate(pk, res, maxDets, recThrs, K):
    """accumulate over the match flags: precision [T, R, K, A, M], recall [T, K, A, M] (-1 where the reference leaves
    -1).  Each maxDet cuts every image to its top detections and mergesorts the category's concatenation, as
    cocoeval.py:317-365 does."""
    flags, npig = res['dt_flags'], res['npig']
    A, T = flags.shape[0], flags.shape[1]
    rt = np.asarray(recThrs, np.float64)
    R, M = rt.size, len(maxDets)
    precision = -np.ones((T, R, K, A, M))
    recall = -np.ones((T, K, A, M))
    dt_off, cpo = pk['dt_off'], pk['cat_pair_off']
    for k in range(K):
        p0, p1 = cpo[k], cpo[k + 1]
        if p0 == p1:
            continue
        i0, i1 = dt_off[p0], dt_off[p1]
        for m, maxDet in enumerate(maxDets):
            sel = np.arange(i0, i1)[pk['dt_rank'][i0:i1] < maxDet]
            inds = np.argsort(-pk['dt_score'][sel], kind='mergesort')
            sel = sel[inds]
            for a in range(A):
                n_pig = int(npig[p0:p1, a].sum())
                if n_pig == 0:
                    continue
                f = flags[a][:, sel]
                dtm, dtIg = (f & 1) != 0, (f & 2) != 0
                tp_sum = np.cumsum(dtm & ~dtIg, axis=1).astype(np.float64)
                fp_sum = np.cumsum(~dtm & ~dtIg, axis=1).astype(np.float64)
                nd = sel.size
                for t in range(T):
                    tp, fp = tp_sum[t], fp_sum[t]
                    rc = tp / n_pig
                    pr = tp / (fp + tp + np.spacing(1))
                    recall[t, k, a, m] = rc[-1] if nd else 0
                    pr = np.maximum.accumulate(pr[::-1])[::-1] if nd else pr
                    ri = np.searchsorted(rc, rt, side='left')
                    bad = np.nonzero(ri >= nd)[0]
                    stop = bad[0] if bad.size else R
                    q = np.zeros(R)
                    q[:stop] = pr[ri[:stop]]
                    precision[t, :, k, a, m] = q
    return precision, recall
