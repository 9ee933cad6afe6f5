"""TEST INFRASTRUCTURE ONLY.  A numpy restatement of the reference's IMDB.evaluate_recall (lib/dataset/imdb.py:291-397),
written from its rules rather than its text, for the CPU tests and for GPU tests at sizes the golden file cannot hold.

  images       entries 0 .. num_images-1 of roidb
  GTs          rows with gt_classes > 0 and gt_overlaps.max(axis=1) == 1
  proposals    candidate_boxes[i], or the rows with gt_classes == 0
  areas        (x2 - x1 + 1) * (y2 - y1 + 1) in the box array's own dtype (uint16 wraps, float32 rounds)
  IoU          bbox_overlaps_cython in float64 (+1 extents; 0 unless iw > 0 and ih > 0; a zero union raises)
  matching     min(#proposals, #GTs) rounds: column maxima over unused rows (lowest row on ties), the largest of them
               (lowest column on ties), recorded; row and column retired.  No proposals: the image adds nothing.
  statistics   recall[t] = count(>= t) / float(num_pos), ar = recalls.mean(); proposal histogram over ranges 1 .. 6

Errors are ValueError where the reference asserts, divides by zero or indexes past its inputs."""
import numpy as np

NAMES = ['all', '0-25', '25-50', '50-100', '100-200', '200-300', '300-inf']
RANGES = [[0 ** 2, 1e5 ** 2], [0 ** 2, 25 ** 2], [25 ** 2, 50 ** 2], [50 ** 2, 100 ** 2], [100 ** 2, 200 ** 2],
          [200 ** 2, 300 ** 2], [300 ** 2, 1e5 ** 2]]


def area(b):
    return (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1)


def iou(boxes, gts):
    """[n, k] float64 overlaps with bbox_overlaps_cython's arithmetic and branches."""
    b = boxes.astype(np.float64)[:, None, :]
    q = gts.astype(np.float64)[None, :, :]
    iw = np.where(q[..., 2] < b[..., 2], q[..., 2], b[..., 2]) - np.where(q[..., 0] > b[..., 0], q[..., 0], b[..., 0]) + 1
    ih = np.where(q[..., 3] < b[..., 3], q[..., 3], b[..., 3]) - np.where(q[..., 1] > b[..., 1], q[..., 1], b[..., 1]) + 1
    inter = iw * ih
    ua = (b[..., 2] - b[..., 0] + 1) * (b[..., 3] - b[..., 1] + 1) + area(gts.astype(np.float64))[None, :] - inter
    hit = (iw > 0) & (ih > 0)
    if np.any(hit & (ua == 0)):
        raise ValueError("zero union")
    out = np.zeros(inter.shape)
    out[hit] = inter[hit] / ua[hit]
    return out


def greedy(ov):
    """The recorded overlap of each round, then zeros up to the GT count."""
    n, k = ov.shape
    rec = np.zeros(k)
    used_r, used_c = np.zeros(n, bool), np.zeros(k, bool)
    for j in range(min(n, k)):
        sub = np.where(used_r[:, None] | used_c[None, :], -np.inf, ov)
        col_max = np.where(used_c, -np.inf, sub.max(axis=0))
        c = int(np.argmax(col_max))
        best = col_max[c]
        if not best >= 0:
            raise ValueError("negative best overlap")
        r = int(np.argmax(sub[:, c]))
        rec[j] = best
        used_r[r] = used_c[c] = True
    return rec


def evaluate(roidb, candidate_boxes=None, thresholds=None, num_images=None):
    """(text, arrays): the returned string and recalls [7, T], ar [7], num_pos [7], gt_overlaps (7 sorted arrays),
    area_counts [6]."""
    n_img = len(roidb) if num_images is None else num_images
    if n_img > len(roidb) or (candidate_boxes is not None and n_img > len(candidate_boxes)):
        raise ValueError("index past the inputs")
    props, gts = [], []
    for i in range(n_img):
        r = roidb[i]
        keep = (r['gt_classes'] > 0) & (r['gt_overlaps'].max(axis=1) == 1)
        gts.append(r['boxes'][keep])
        props.append(r['boxes'][r['gt_classes'] == 0] if candidate_boxes is None else candidate_boxes[i])
    counts = [sum(int(((area(p) >= lo) & (area(p) < hi)).sum()) for p in props) for lo, hi in RANGES[1:]]
    total = float(sum(counts))
    if total == 0:
        raise ValueError("no proposal in any range")
    lines = ['percentage of {} {}'.format(nm, c / total) for nm, c in zip(NAMES[1:], counts)]
    lines.append('average number of proposal {}'.format(total / n_img))
    thr = np.arange(0.5, 0.95 + 1e-5, 0.05) if thresholds is None else np.asarray(thresholds, np.float64)
    out = dict(recalls=[], ar=[], num_pos=[], gt_overlaps=[], area_counts=np.asarray(counts, np.int64))
    for nm, (lo, hi) in zip(NAMES, RANGES):
        vals, num_pos = [], 0
        for p, g in zip(props, gts):
            a = area(g)
            g = g[(a >= lo) & (a < hi)]
            num_pos += g.shape[0]
            if p.shape[0] == 0:
                continue
            vals.append(greedy(iou(p[:, :4], g[:, :4])) if g.shape[0] else np.zeros(0))
        ov = np.sort(np.concatenate(vals)) if vals else np.zeros(0)
        with np.errstate(invalid='ignore', divide='ignore'):
            rc = np.array([(ov >= t).sum() / float(num_pos) for t in thr], np.float64).reshape(-1)
            ar = rc.mean() if rc.size else np.float64(np.nan)
        lines.append('average recall for {}: {:.3f}'.format(nm, ar))
        lines += ['recall @{:.2f}: {:.3f}'.format(t, x) for t, x in zip(thr, rc)]
        out['recalls'].append(rc)
        out['ar'].append(ar)
        out['num_pos'].append(num_pos)
        out['gt_overlaps'].append(ov)
    out['recalls'] = np.array(out['recalls']).reshape(len(NAMES), thr.size)
    out['ar'] = np.array(out['ar'], np.float64)
    out['num_pos'] = np.array(out['num_pos'], np.int64)
    return ''.join(lines), out
