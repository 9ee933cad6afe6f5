"""Proposal recall of a roidb: IMDB.evaluate_recall of the reference (lib/dataset/imdb.py:291-397), with the greedy
matching, the recalls and the proposal histogram on the device (csrc/proposal_recall.cu, ops.proposal_recall).

What the host does, in the reference's own numpy expressions: pick each image's GTs (gt_classes > 0 and max
gt_overlaps == 1) and proposals (candidate_boxes[i], or the roidb's gt_classes == 0 rows), and compute the GT area
ranges in the box array's own dtype.  uint16 boxes (coco.gt_roidb, PascalVOC.gt_roidb) wrap their area modulo 65536
as the reference's do, so a 300 x 300 GT counts in 100-200; float32 areas round in float32."""
import numpy as np

from . import ops

AREA_NAMES = ['all', '0-25', '25-50', '50-100', '100-200', '200-300', '300-inf']
AREA_RANGES = [[0 ** 2, 1e5 ** 2], [0 ** 2, 25 ** 2], [25 ** 2, 50 ** 2], [50 ** 2, 100 ** 2], [100 ** 2, 200 ** 2],
               [200 ** 2, 300 ** 2], [300 ** 2, 1e5 ** 2]]


def default_thresholds():
    """IoU 0.50:0.05:0.95 with the values numpy gives (0.6000000000000001, ...)."""
    return np.arange(0.5, 0.95 + 1e-5, 0.05)


def _areas(b):
    return (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1)


def recall_inputs(roidb, candidate_boxes=None, num_images=None):
    """The CSR inputs of ops.proposal_recall: (prop_box, prop_off, gt_box, gt_off, gt_range)."""
    n_img = len(roidb) if num_images is None else int(num_images)
    if n_img > len(roidb):
        raise ValueError("evaluate_recall: %d images, but the roidb has %d entries" % (n_img, len(roidb)))
    if candidate_boxes is not None and n_img > len(candidate_boxes):
        raise ValueError("evaluate_recall: %d images, but candidate_boxes has %d entries"
                         % (n_img, len(candidate_boxes)))
    props, gts, masks = [], [], []
    for i in range(n_img):
        r = roidb[i]
        boxes = np.asarray(r['boxes'])
        gt_classes = np.asarray(r['gt_classes'])
        max_gt_overlaps = np.asarray(r['gt_overlaps']).max(axis=1)
        g = boxes[np.where((gt_classes > 0) & (max_gt_overlaps == 1))[0], :]
        a = _areas(g)
        mask = np.zeros(g.shape[0], np.uint8)
        for k, (lo, hi) in enumerate(AREA_RANGES):
            mask |= (((a >= lo) & (a < hi)).astype(np.uint8) << k)
        p = boxes[np.where(gt_classes == 0)[0], :] if candidate_boxes is None else np.asarray(candidate_boxes[i])
        if p.ndim != 2 or p.shape[1] < 4 or g.ndim != 2 or g.shape[1] < 4:
            raise ValueError("evaluate_recall: image %d: boxes must be [n, >= 4] arrays" % i)
        props.append(p[:, :4])
        gts.append(g[:, :4].astype(np.float64))
        masks.append(mask)
    dtypes = {p.dtype for p in props if p.shape[0]}
    if len(dtypes) > 1:
        raise ValueError("evaluate_recall: the proposals mix dtypes %s; their areas are computed in their own dtype"
                         % sorted(str(d) for d in dtypes))
    dt = dtypes.pop() if dtypes else np.dtype(np.float32)
    prop_off = np.zeros(n_img + 1, np.int64)
    np.cumsum([p.shape[0] for p in props], out=prop_off[1:])
    gt_off = np.zeros(n_img + 1, np.int64)
    np.cumsum([g.shape[0] for g in gts], out=gt_off[1:])
    prop_box = np.concatenate([p.astype(dt, copy=False) for p in props]) if n_img else np.zeros((0, 4), dt)
    gt_box = np.concatenate(gts) if n_img else np.zeros((0, 4))
    gt_range = np.concatenate(masks) if n_img else np.zeros(0, np.uint8)
    if prop_off[-1] >= 2 ** 31 or gt_off[-1] >= 2 ** 31:
        raise ValueError("evaluate_recall: more than 2^31 - 1 proposals or GTs")
    return prop_box, prop_off, gt_box, gt_off, gt_range


def recall_text(res, thresholds):
    """The lines evaluate_recall prints, in order, from ops.proposal_recall's results."""
    lines = []
    total_counts = float(sum(int(c) for c in res['area_counts']))
    if total_counts == 0:
        raise ValueError("evaluate_recall: no proposal has an area in any range (the reference divides by zero)")
    for name, count in zip(AREA_NAMES[1:], res['area_counts']):
        lines.append('percentage of {} {}'.format(name, int(count) / total_counts))
    lines.append('average number of proposal {}'.format(float(res['avg_proposals'])))
    for r, name in enumerate(AREA_NAMES):
        lines.append('average recall for {}: {:.3f}'.format(name, res['ar'][r]))
        for threshold, recall in zip(thresholds, res['recalls'][r]):
            lines.append('recall @{:.2f}: {:.3f}'.format(threshold, recall))
    return lines


def evaluate_recall(roidb, candidate_boxes=None, thresholds=None, num_images=None, device="cuda", verbose=True):
    """Proposal recall per GT area range, as the reference's IMDB.evaluate_recall: for every GT, the IoU of the
    proposal that greedily covers it, then the recall at each IoU threshold (default 0.50:0.05:0.95) and the average
    recall, per area range, and the share of proposals in each range.  Prints the lines and returns them concatenated
    without separators, as the reference's code does under Python 3 (Python 2's 12-digit str(float) of the percentages
    is not reproduced).  num_images: the images scored, entries 0 .. num_images-1 (default: all of roidb).  Raises
    ValueError where the reference would assert (a negative best overlap), divide by zero or index past its inputs."""
    thr = default_thresholds() if thresholds is None else np.asarray(thresholds)
    if thr.ndim != 1 or thr.dtype != np.float64:
        raise ValueError("evaluate_recall: thresholds must be a 1-D array-like of floats (float64)")
    prop_box, prop_off, gt_box, gt_off, gt_range = recall_inputs(roidb, candidate_boxes, num_images)
    res = ops.proposal_recall(prop_box, prop_off, gt_box, gt_off, gt_range, thr, device=device)
    lines = recall_text(res, thr)
    if verbose:
        for line in lines:
            print(line)
    return ''.join(lines)
