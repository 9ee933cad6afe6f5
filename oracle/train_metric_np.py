"""float64 numpy restatement of the training metrics' per-step updates (lib/train_utils/metric.py:50-95, 104-300) on
this package's tensor layouts, in the accumulator form of csrc/train_metric.cu: (num_inst[8], sum_metric[8]) in the
slot order of sniper_b200.metric.SLOTS.  p[label] + 1e-14 is rounded to float32 as the reference's `cls += 1e-14` does;
the log and the sums are float64 (the reference takes both in float32)."""
import numpy as np


def _terms(p2, lab):
    """p2 [n, 2] or [n, K] float32 rows, lab [n] int: (hits, log-loss sum, count) over rows with lab != -1."""
    keep = lab != -1
    p, l = p2[keep], lab[keep]
    hits = int(np.sum(np.argmax(p, axis=1) == l))
    sel = (p[np.arange(len(l)), l] + np.float32(1e-14)).astype(np.float32)
    return hits, float(np.sum(-np.log(sel.astype(np.float64)))), int(keep.sum())


def two_way_rows(prob, A):
    """NHWC [B,H,W,>=2A] (bg = channel a, fg = A+a) -> [B*A*H*W, 2] rows in the labels' (b, a, h, w) order."""
    B, H, W = prob.shape[:3]
    p = prob[..., :2 * A].reshape(B, H, W, 2, A).transpose(0, 4, 1, 2, 3)
    return np.ascontiguousarray(p.reshape(-1, 2))


def step(rpn_prob, rpn_label, A, cls_prob, cls_label, rpn_l1, rcnn_l1, af_prob=None, af_label=None):
    """One step's contribution: (num_inst int64 [8], sum_metric float64 [8]); rpn_l1 / rcnn_l1 are the step's
    smooth-L1 loss sums (loss_buf[1] / [3])."""
    num = np.zeros(8, np.int64)
    s = np.zeros(8, np.float64)
    h, ll, n = _terms(two_way_rows(rpn_prob, A), np.asarray(rpn_label).astype(np.int32).reshape(-1))
    num[0:3] = n
    s[0], s[1], s[2] = h, ll, float(np.float32(rpn_l1))
    h, ll, n = _terms(np.asarray(cls_prob, np.float32), np.asarray(cls_label).astype(np.int32).reshape(-1))
    num[3:6] = n
    s[3], s[4], s[5] = h, ll, float(np.float32(rcnn_l1))
    if af_prob is not None:
        h, ll, n = _terms(two_way_rows(af_prob, 1), np.asarray(af_label).astype(np.int32).reshape(-1))
        num[6:8] = n
        s[6], s[7] = h, ll
    return num, s
