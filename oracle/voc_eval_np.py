"""Float64 numpy restatement of the reference's PASCAL VOC evaluation (lib/dataset/pascal_voc_eval.py:39-181) on the
inputs csrc/voc_eval.cu takes: detections class-major in the host's sorted order, GTs a CSR over the (class, image)
pairs.  The per-detection loop is the reference's; numpy's pairwise summation, which np.sum runs in voc_ap, is written
out (pairwise_sum) so that the order the device reproduces is stated in one place."""
import numpy as np


def match(det_box, det_pair, gt_box, gt_difficult, gt_off, thresholds):
    """flags [T, N] uint8 (1 tp, 2 fp, 0 a hit on a difficult GT), one detection at a time in sorted order."""
    det_box = np.asarray(det_box, np.float64).reshape(-1, 4)
    gt_box = np.asarray(gt_box, np.float64).reshape(-1, 4)
    gt_difficult = np.asarray(gt_difficult).astype(bool)
    thresholds = np.asarray(thresholds, np.float64).reshape(-1)
    flags = np.zeros((thresholds.size, len(det_box)), np.uint8)
    for t, ovthresh in enumerate(thresholds):
        det = {}
        for d in range(len(det_box)):
            p = int(det_pair[d])
            g0, g1 = int(gt_off[p]), int(gt_off[p + 1])
            bb = det_box[d]
            bbgt = gt_box[g0:g1]
            ovmax = -np.inf
            if bbgt.size > 0:
                ixmin = np.maximum(bbgt[:, 0], bb[0])
                iymin = np.maximum(bbgt[:, 1], bb[1])
                ixmax = np.minimum(bbgt[:, 2], bb[2])
                iymax = np.minimum(bbgt[:, 3], bb[3])
                iw = np.maximum(ixmax - ixmin + 1., 0.)
                ih = np.maximum(iymax - iymin + 1., 0.)
                inters = iw * ih
                uni = ((bb[2] - bb[0] + 1.) * (bb[3] - bb[1] + 1.) +
                       (bbgt[:, 2] - bbgt[:, 0] + 1.) * (bbgt[:, 3] - bbgt[:, 1] + 1.) - inters)
                with np.errstate(divide='ignore', invalid='ignore'):
                    overlaps = inters / uni
                ovmax = np.max(overlaps)
                jmax = np.argmax(overlaps)
            f = 2
            if ovmax > ovthresh:
                taken = det.setdefault(p, np.zeros(g1 - g0, bool))
                if gt_difficult[g0 + jmax]:
                    f = 0
                elif not taken[jmax]:
                    f = 1
                    taken[jmax] = True
            flags[t, d] = f
    return flags


def pairwise_sum(a):
    """np.sum of a contiguous float64 array: 0. + pairwise_sum (numpy/_core/src/umath/loops_utils.h.src)."""
    def pw(lo, n):
        if n < 8:
            res = 0.
            for i in range(n):
                res = res + a[lo + i]
            return res
        if n <= 128:
            r = [a[lo + j] for j in range(8)]
            i = 8
            while i < n - (n % 8):
                for j in range(8):
                    r[j] = r[j] + a[lo + i + j]
                i += 8
            res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
            while i < n:
                res = res + a[lo + i]
                i += 1
            return res
        n2 = n // 2
        n2 -= n2 % 8
        return pw(lo, n2) + pw(lo + n2, n - n2)
    a = np.asarray(a, np.float64)
    return np.float64(0.) + np.float64(pw(0, a.size))


def voc_ap(rec, prec, use_07_metric=False, thresholds_07=None):
    """voc_ap (pascal_voc_eval.py:39-70) with the area metric's sum written as pairwise_sum."""
    if use_07_metric:
        ap = 0.
        for t in (np.arange(0., 1.1, 0.1) if thresholds_07 is None else thresholds_07):
            with np.errstate(invalid='ignore'):
                sel = rec >= t
            p = 0 if np.sum(sel) == 0 else np.max(prec[sel])
            ap += p / 11.
        return np.float64(ap)
    mrec = np.concatenate(([0.], rec, [1.]))
    mpre = np.concatenate(([0.], prec, [0.]))
    for i in range(mpre.size - 1, 0, -1):
        mpre[i - 1] = np.maximum(mpre[i - 1], mpre[i])
    i = np.where(mrec[1:] != mrec[:-1])[0]
    with np.errstate(invalid='ignore'):
        return pairwise_sum((mrec[i + 1] - mrec[i]) * mpre[i + 1])


def accumulate(flags, det_off, npos, use_07_metric, thresholds_07=None):
    """rec, prec [T, N] and ap [T, C] from match's flags (pascal_voc_eval.py:173-179)."""
    T, N = flags.shape
    C = len(det_off) - 1
    rec, prec = np.zeros((T, N)), np.zeros((T, N))
    ap = np.zeros((T, C))
    for t in range(T):
        for c in range(C):
            a, b = int(det_off[c]), int(det_off[c + 1])
            f = flags[t, a:b]
            tp = np.cumsum((f == 1).astype(np.float64))
            fp = np.cumsum((f == 2).astype(np.float64))
            with np.errstate(divide='ignore', invalid='ignore'):
                r = tp / float(npos[c])
            p = tp / np.maximum(tp + fp, np.finfo(np.float64).eps)
            rec[t, a:b], prec[t, a:b] = r, p
            ap[t, c] = voc_ap(r, p, use_07_metric, thresholds_07)
    return rec, prec, ap
