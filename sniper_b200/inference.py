"""Post-processing of the multi-scale inference path (the half of lib/inference.py that is arithmetic rather than
bookkeeping): per-chip box decoding (`Tester.detect`, :100-139), score thresholding (`get_detections`, :291-301) and the
cross-scale aggregation with per-(image, class) soft-NMS (`Tester.aggregate`, :152-230).

Two detection backends feed the aggregation; they differ only in where rows are decoded and thresholded.  The host one
(`detect_postprocess`, `threshold_detections`, nested lists per class / image / chip) is the reference's arithmetic in
numpy and the oracle of the other.  The device one keeps every detection on the GPU: `ops.detect_post` appends each
batch's surviving rows with their `pack_key` order key to a `DeviceDetections` run buffer.

`aggregate` reduces either to float32 rows and an (image, class) problem index per scale, and from there has one path:
a stable sort by problem, segment offsets, the soft-NMS, the MAX_PER_IMAGE cut.  The reference farms the NMS out to
`Pool(32)` processes, one `cpu_soft_nms` call per image and class; here every problem of the run is ONE launch of
`sniper_soft_nms_batched`.  `backend="host"` runs the C-ABI host `sniper_cpu_soft_nms` (bit-identical to the
reference's Cython) per problem instead -- the parity tests compare the two.
Not built (needs OpenCV, absent from this image): FocusChip generation
(`lib/chips/chips_inference.py`: cv2.dilate + findContours).
"""
import numpy as np
import torch

from . import host, ops
from ._lib import SniperError as _SniperError


def bbox_pred(boxes, box_deltas):
    """nonlinear_pred (lib/bbox/bbox_transform.py:93-133): class-agnostic rois [N,4] + deltas [N,4k] -> boxes [N,4k],
    float64 like the reference (`boxes.astype(np.float)`)."""
    if boxes.shape[0] == 0:
        return np.zeros((0, box_deltas.shape[1]))
    boxes = boxes.astype(float, copy=False)
    w = boxes[:, 2] - boxes[:, 0] + 1.0
    h = boxes[:, 3] - boxes[:, 1] + 1.0
    cx = boxes[:, 0] + 0.5 * (w - 1.0)
    cy = boxes[:, 1] + 0.5 * (h - 1.0)
    pcx = box_deltas[:, 0::4] * w[:, None] + cx[:, None]
    pcy = box_deltas[:, 1::4] * h[:, None] + cy[:, None]
    pw = np.exp(box_deltas[:, 2::4]) * w[:, None]
    ph = np.exp(box_deltas[:, 3::4]) * h[:, None]
    out = np.zeros(box_deltas.shape)
    out[:, 0::4] = pcx - 0.5 * (pw - 1.0)
    out[:, 1::4] = pcy - 0.5 * (ph - 1.0)
    out[:, 2::4] = pcx + 0.5 * (pw - 1.0)
    out[:, 3::4] = pcy + 0.5 * (ph - 1.0)
    return out


def clip_boxes(boxes, im_shape):
    boxes[:, 0::4] = np.maximum(np.minimum(boxes[:, 0::4], im_shape[1] - 1), 0)
    boxes[:, 1::4] = np.maximum(np.minimum(boxes[:, 1::4], im_shape[0] - 1), 0)
    boxes[:, 2::4] = np.maximum(np.minimum(boxes[:, 2::4], im_shape[1] - 1), 0)
    boxes[:, 3::4] = np.maximum(np.minimum(boxes[:, 3::4], im_shape[0] - 1), 0)
    return boxes


def detect_postprocess(rois, cls_prob, bbox_deltas, im_info, batch_size):
    """Tester.detect :113-131 for one device's outputs: rois [B*R,5] (batch_idx, x1..y2), cls_prob [B*R,K], bbox_deltas
    [B*R,4], im_info [B,3] -> per chip (scores [R,K], boxes [R,4] in image scale)."""
    rois, cls_prob = np.asarray(rois), np.asarray(cls_prob)
    bbox_deltas, im_info = np.asarray(bbox_deltas), np.asarray(im_info)
    scores, preds = [], []
    for idx in range(batch_size):
        cids = np.where(rois[:, 0] == idx)[0]
        cboxes = clip_boxes(bbox_pred(rois[cids, 1:], bbox_deltas[cids]), im_info[idx, :2])
        preds.append(cboxes / im_info[idx, 2])
        scores.append(cls_prob[cids])
    return scores, preds


def threshold_detections(cscores, cboxes, num_classes, cls_thresh=1e-3, prune=None):
    """get_detections :291-301: per class j >= 1 the rows with score > cls_thresh as [n,5] (x1,y1,x2,y2,score).
    prune = (chip [x1,y1,x2,y2], im_width, im_height): additionally the `do_pruning` step (:335-351) -- rows moved to image
    coordinates and detections cut by a chip border dropped (chips_inference.project_and_prune), on all classes at once."""
    # one pass over the [R, K] score matrix instead of K np.where calls: (class, roi) pairs in class-major, roi-minor
    # order = the order the per-class loop of the reference produces
    cls_idx, roi_idx = np.nonzero(cscores[:, 1:num_classes].T > cls_thresh)
    rows = np.empty((len(roi_idx), 5), np.float32)
    rows[:, :4] = cboxes[roi_idx, 0:4]
    rows[:, 4] = cscores[roi_idx, cls_idx + 1]
    if prune is not None:
        from .chips_inference import prune_mask
        chip, im_w, im_h = prune
        rows = rows.astype(np.float64)
        rows[:, 0] += chip[0]; rows[:, 2] += chip[0]
        rows[:, 1] += chip[1]; rows[:, 3] += chip[1]
        keep = prune_mask(rows, chip, im_w, im_h)
        rows, cls_idx = rows[keep], cls_idx[keep]
    cuts = np.searchsorted(cls_idx, np.arange(1, num_classes - 1))
    return [np.zeros((0, 5), rows.dtype)] + np.split(rows, cuts)


def _valid_range_filter(cls_dets, valid_range):
    """Tester.aggregate :176-186 (areas = (x-extent) * (y-extent), no +1; lower bound exclusive, upper inclusive)."""
    heights = cls_dets[:, 2] - cls_dets[:, 0]
    widths = cls_dets[:, 3] - cls_dets[:, 1]
    areas = widths * heights
    lo = np.where(areas > valid_range[0] * valid_range[0])[0] if valid_range[0] > 0 else np.arange(len(areas))
    hi = np.where(areas <= valid_range[1] * valid_range[1])[0] if valid_range[1] > 0 else np.arange(len(areas))
    return cls_dets[np.intersect1d(lo, hi), :]


# ---------------------------------------------------------------------------------------------
# device detection backend: chip table, order key, run buffer
# ---------------------------------------------------------------------------------------------
CHIP_COLS = 12
_ROI_BITS, _CHIP_BITS, _SCALE_BITS, _CLASS_BITS, _IMAGE_BITS = 16, 14, 4, 10, 19


def pack_key(image, cls, scale, chip, roi):
    """The int64 order key `sniper_detect_post` gives a row: sorting by it groups the (image, class) problems in
    `aggregate`'s order and, inside a problem, stacks rows by scale, chip id and roi as the reference's loops do."""
    image, cls, scale, chip, roi = (np.asarray(v, np.int64) for v in (image, cls, scale, chip, roi))
    return ((((image << _CLASS_BITS | cls) << _SCALE_BITS | scale) << _CHIP_BITS | chip) << _ROI_BITS) | roi


def unpack_key(key):
    """(image, class, scale, chip, roi) of pack_key."""
    key = np.asarray(key, np.int64)
    out = []
    for bits in (_ROI_BITS, _CHIP_BITS, _SCALE_BITS, _CLASS_BITS, _IMAGE_BITS):
        out.append(key & ((1 << bits) - 1))
        key = key >> bits
    return tuple(out[::-1])


def chip_table(roidb, im_ids, chip_ids, do_pruning, valid_range, seen=None):
    """The per-chip table of one batch for `ops.detect_post`: float64 [B, 12] = image id, chip id, the chip rectangle
    `inference_crops[chip]` in image coordinates, image width and height, the prune flag, the scale's valid range and
    one unused column.  A (image, chip) pair already in the set `seen` (the iterator repeats chips to fill its last
    batch) gets image id -1 and emits nothing, as the host path overwrites the same list cell; new pairs are added."""
    t = np.zeros((len(im_ids), CHIP_COLS), np.float64)
    for k, (im, chip) in enumerate(zip(im_ids, chip_ids)):
        im, chip = int(im), int(chip)
        if not (0 <= im < (1 << _IMAGE_BITS) and 0 <= chip < (1 << _CHIP_BITS)):
            raise ValueError("chip_table: image %d / chip %d do not fit the order key" % (im, chip))
        r = roidb[im]
        t[k, 0], t[k, 1] = im, chip
        t[k, 2:6] = np.asarray(r['inference_crops'][chip], np.float64)[:4]
        t[k, 6], t[k, 7] = r['width'], r['height']
        t[k, 8] = 1.0 if do_pruning else 0.0
        t[k, 9], t[k, 10] = valid_range[0], valid_range[1]
        if seen is not None:
            if (im, chip) in seen:
                t[k, 0] = -1.0
            seen.add((im, chip))
    return t


class DeviceDetections(object):
    """The detections of one test scale on the device: rows [n, 5] float32 (x1, y1, x2, y2, score) and their int64
    order keys, appended batch by batch by `ops.detect_post` at a device-side cursor.

    Capacity policy: a batch can add at most B * R * (K - 1) rows, and a launch is only issued when the buffer can
    take that on top of an upper bound of the cursor.  The bound is the last cursor value read back (a non-blocking
    copy into pinned memory after every launch, polled through its event, so it lags by the batches still in flight)
    plus the worst case of every launch since; the current batch never waits.  When the bound does not fit, a growable
    buffer is reallocated (doubled at least) and the rows copied over on the stream; a fixed one (`growable=False`)
    refuses the batch with a `SniperError`.  No row is ever dropped: should a launch find its rows not fitting after
    all, it writes none, records the count, and `finish()` raises."""

    def __init__(self, device="cuda", capacity=1 << 18, growable=True):
        self.device = torch.device(device)
        self.growable = growable
        self.rows = torch.empty(int(capacity), 5, device=self.device)
        self.keys = torch.empty(int(capacity), dtype=torch.int64, device=self.device)
        self.state = torch.zeros(2, dtype=torch.int64, device=self.device)
        self.workspace = ops.detect_post_workspace(self.device)
        self._known = 0            # the cursor after the last launch whose read-back has arrived
        self._inflight = []        # (event, pinned copy of state, worst case of that launch), oldest first
        self._n = None

    @property
    def capacity(self):
        return self.rows.shape[0]

    def rows_bound(self):
        while self._inflight and self._inflight[0][0].query():
            self._known = int(self._inflight.pop(0)[1][0])
        return self._known + sum(w for _, _, w in self._inflight)

    def append(self, rois, cls_prob, bbox_pred, im_info, chips, cls_thresh=1e-3, scale=0):
        """One batch: the network's output tensors and the batch's `chip_table` (host array or device tensor)."""
        self._n = None
        worst = rois.shape[0] * (cls_prob.shape[1] - 1)
        bound = self.rows_bound()
        if self.growable and bound + worst > self.capacity:
            cap = max(2 * self.capacity, bound + worst)
            rows = torch.empty(cap, 5, device=self.device)
            keys = torch.empty(cap, dtype=torch.int64, device=self.device)
            rows[:bound].copy_(self.rows[:bound])
            keys[:bound].copy_(self.keys[:bound])
            self.rows, self.keys = rows, keys
        if not torch.is_tensor(chips):
            chips = torch.from_numpy(np.ascontiguousarray(chips, np.float64)).to(self.device, non_blocking=True)
        ops.detect_post(rois, cls_prob, bbox_pred, im_info, chips, self.rows, self.keys, self.state, self.workspace,
                        cls_thresh=cls_thresh, scale=scale, rows_bound=bound)
        host = torch.empty(2, dtype=torch.int64, pin_memory=True)
        host.copy_(self.state, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._inflight.append((ev, host, worst))

    def finish(self):
        """Waits for the launches so far and returns the number of rows held."""
        if self._n is None:
            state = self.state.cpu()
            self._inflight, self._known = [], int(state[0])
            if int(state[1]):
                raise _SniperError("detect_post: a batch needed %d rows in a run buffer of %d; its rows were not "
                                   "written" % (int(state[1]), self.capacity))
            self._n = self._known
        return self._n

    def __len__(self):
        return self.finish()

    def result(self):
        """(rows [n,5], keys [n]) views of the run so far (waits)."""
        n = self.finish()
        return self.rows[:n], self.keys[:n]


def _run_problems(dets, num_classes):
    """One scale's `DeviceDetections` -> (rows [n,5], int64 problem index image * (K - 1) + class - 1 [n]) on its
    device, sorted by key: image, class, chip, roi."""
    rows, keys = dets.result()
    keys, order = torch.sort(keys, stable=True)
    shift = _ROI_BITS + _CHIP_BITS + _SCALE_BITS
    cls = (keys >> shift) & ((1 << _CLASS_BITS) - 1)
    return rows[order], (keys >> (shift + _CLASS_BITS)) * (num_classes - 1) + cls - 1


def _list_problems(all_cls_dets, valid_range, num_images, num_classes, device):
    """One scale's nested lists all_cls_dets[j][i][chip] -> (rows [n,5], int64 problem index [n]) on `device`, stacked
    class by class, image by image, chip by chip, through the scale's valid range (the area rule of
    `_valid_range_filter`)."""
    blocks, prob = [np.zeros((0, 5), np.float32)], [0]
    for j in range(1, num_classes):
        for i in range(num_images):
            for cls_dets in all_cls_dets[j][i]:
                blocks.append(np.asarray(cls_dets, np.float32).reshape(-1, 5))
                prob.append(i * (num_classes - 1) + j - 1)
    d = np.concatenate(blocks, 0)
    p = np.repeat(np.array(prob, np.int64), [len(b) for b in blocks])
    areas = (d[:, 3] - d[:, 1]) * (d[:, 2] - d[:, 0])
    keep = np.ones(len(d), bool)
    if valid_range[0] > 0:
        keep &= areas > valid_range[0] * valid_range[0]
    if valid_range[1] > 0:
        keep &= areas <= valid_range[1] * valid_range[1]
    return torch.from_numpy(d[keep]).to(device), torch.from_numpy(p[keep]).to(device)


def aggregate(scale_cls_dets, valid_ranges, num_images, num_classes, sigma=0.55, nms_thresh=0.3, max_per_image=100,
              backend="device", device="cuda"):
    """Tester.aggregate (:152-230).  scale_cls_dets[s][j][i] = list over chips of [n,5] detections of class j in image i
    at scale s, or one `DeviceDetections` per scale (its rows passed the valid range in `ops.detect_post`).  Returns
    all_boxes[j][i] = [n,5] after the valid-range filter, Gaussian soft-NMS (sigma, threshold 0.001; nms_worker ->
    nms_wrapper -> cpu_soft_nms) and the MAX_PER_IMAGE cut.
    Every scale's rows are tagged with their (image, class) problem; one stable sort by problem then stacks a problem's
    rows in the (scale, chip, row) order of the reference's nested loops.  The sort runs where the rows are: on the
    device for `DeviceDetections`, or for nested lists with backend="device"; on the CPU otherwise."""
    assert len(scale_cls_dets) == len(valid_ranges), 'A valid range should be specified for each test scale'
    on_device = [isinstance(d, DeviceDetections) for d in scale_cls_dets]
    if any(on_device):
        if not all(on_device):
            raise TypeError("aggregate: every scale's detections must come from the same backend (got nested lists "
                            "and DeviceDetections)")
        parts = [_run_problems(d, num_classes) for d in scale_cls_dets]
    else:
        dev = device if backend == "device" else "cpu"
        parts = [_list_problems(d, vr, num_images, num_classes, dev) for d, vr in zip(scale_cls_dets, valid_ranges)]
    prob, order = torch.sort(torch.cat([p for _, p in parts]), stable=True)
    rows = torch.cat([r for r, _ in parts], 0)[order]
    nprob = num_images * (num_classes - 1)
    if rows.shape[0] and (int(prob[0]) < 0 or int(prob[-1]) >= nprob):
        raise ValueError("aggregate: detections of an image or class outside %d images x %d classes"
                         % (num_images, num_classes))
    offsets = torch.searchsorted(prob, torch.arange(nprob + 1, device=prob.device)).to(torch.int32)
    if backend == "device" and rows.shape[0]:
        out, counts = ops.soft_nms_batched(rows, offsets, sigma=sigma, Nt=nms_thresh, threshold=0.001, method=2)
        out, counts, offsets = out.cpu().numpy(), counts.cpu().numpy(), offsets.cpu().numpy()
        final = [out[offsets[p]:offsets[p] + counts[p]] for p in range(len(counts))]
    else:
        final = [host.cpu_soft_nms(p.copy(), sigma=sigma, Nt=nms_thresh, threshold=0.001, method=2) if len(p) else p
                 for p in np.split(rows.cpu().numpy(), offsets.cpu().numpy()[1:-1])]
    return _per_image(final, num_images, num_classes, max_per_image)


def _per_image(final, num_images, num_classes, max_per_image):
    """final[i * (num_classes - 1) + j - 1] -> all_boxes[j][i] with the MAX_PER_IMAGE cut (Tester.aggregate :202-214)."""
    all_boxes = [[[] for _ in range(num_images)] for _ in range(num_classes)]
    for i in range(num_images):
        for j in range(1, num_classes):
            all_boxes[j][i] = final[i * (num_classes - 1) + (j - 1)]
    for i in range(num_images):
        if max_per_image > 0:
            image_scores = np.hstack([all_boxes[j][i][:, -1] for j in range(1, num_classes)])
            if len(image_scores) > max_per_image:
                image_thresh = np.sort(image_scores)[-max_per_image]
                for j in range(1, num_classes):
                    keep = np.where(all_boxes[j][i][:, -1] >= image_thresh)[0]
                    all_boxes[j][i] = all_boxes[j][i][keep, :]
    return all_boxes
