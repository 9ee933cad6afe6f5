"""TEST INFRASTRUCTURE ONLY.  numpy restatement of the reference's proposal NMS `nmsp` (lib/nms/nms.py:48-80, IoU
threshold 0.7) with the tie rule of the device kernel (sniper_proposal_nms_batched) made explicit: the rows are visited
in descending score order and exact ties go to the higher input row, which is `scores.argsort()[::-1]` wherever
numpy's argsort is stable.  The reference's own `argsort()` (quicksort) leaves the order of ties to the platform; on
tie-free inputs the two agree (tests/golden/proposals_ref.npz holds the reference's results).  The arithmetic is
nmsp's: float32 throughout for float32 input."""
import numpy as np

THRESH = 0.7


def nmsp_keep(dets):
    """Kept row indices (int64 array) of dets [N, 5] float32 (x1, y1, x2, y2, score), in keep order."""
    if dets.shape[0] == 0:
        return np.zeros(0, dtype=np.int64)
    x1, y1, x2, y2, scores = dets[:, 0], dets[:, 1], dets[:, 2], dets[:, 3], dets[:, 4]
    areas = (x2 - x1 + 1) * (y2 - y1 + 1)
    order = np.argsort(scores, kind="stable")[::-1]
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(i)
        xx1 = np.maximum(x1[i], x1[order[1:]])
        yy1 = np.maximum(y1[i], y1[order[1:]])
        xx2 = np.minimum(x2[i], x2[order[1:]])
        yy2 = np.minimum(y2[i], y2[order[1:]])
        w = np.maximum(0.0, xx2 - xx1 + 1)
        h = np.maximum(0.0, yy2 - yy1 + 1)
        inter = w * h
        ovr = inter / (areas[i] + areas[order[1:]] - inter)
        order = order[np.where(ovr <= THRESH)[0] + 1]
    return np.array(keep, dtype=np.int64)
