"""Host-side SNIPER chip sampling for one roidb entry: positive chips per scale, box -> chip assignment, negative-chip
mining.  Same class / method names, inputs and outputs as the reference's `chip_worker`
(lib/data_utils/data_workers.py:373-594) so that lib/iterators/MNIteratorBase.py can call it unchanged:

    w = chip_worker(cfg, chip_size)          # cfg.TRAIN.{VALID_RANGES, SCALES, CPP_CHIPS, USE_NEG_CHIPS}
    r['crops'] = w.chip_extractor(r)         # [[chip xyxy (float64, image coords), im_scale, h, w, scale_idx], ...]
    props, neg_chips, neg_props = w.box_assigner(r)

Stays on the host (north_star: "lib/chips positive/negative chip sampling ... stay on host"); the greedy cover itself
is the C-ABI call `sniper_chips_generate` (csrc/host_ops.cpp, bit-exact vs lib/chips/cchips.cpp) and the box/chip
containment matrix is `sniper_bbox_overlaps(ignore=1)` (lib/bbox/bbox.pyx:59-95).  The per-box Python loops of the
reference are expressed as array operations here; every comparison is made on the same float64 values in the same
direction, so the returned indices are identical (tests/test_chip_worker_cpu.py runs the reference class itself)."""
import numpy as np

from . import host


def image_scales(scales, width, height):
    """The scaling factor of every entry of TRAIN.SCALES for one image (data_workers.py:408-426 / :466-484).
    Resolution mode ((min_side, max_side) pairs): min_side / shorter side, capped so that round(scale * longer side)
    stays <= max_side; a non-positive min_side means "fit the longer side".  Factor mode (floats): as given, except
    that the LAST entry is the longer side in pixels."""
    longer, shorter = max(width, height), min(width, height)
    res_based = isinstance(scales[0], (list, tuple))
    out = []
    for i, s in enumerate(scales):
        if res_based:
            lo, hi = s[0], s[1]
            if lo > 0:
                f = float(lo) / float(shorter)
                if hi > 0 and np.round(f * longer) > hi:
                    f = float(hi) / float(longer)
            else:
                f = float(hi) / float(longer)
        else:
            f = s / float(longer) if i == len(scales) - 1 else s
        out.append(f)
    return out


class chip_generator(object):
    """lib/chips/chip_generator.py:10-27 (`use_cpp` path): boxes already multiplied by the scale, clipped in float64 by
    `clip_boxes(boxes, [height-1, width-1])` -- i.e. to [0, width-2] x [0, height-2], bbox_transform.py:35-50 subtracts
    one more -- and only then narrowed to float32 for chips::cgenerate."""

    def __init__(self, chip_stride=32, use_cpp=True):
        self.chip_stride = chip_stride
        self.use_cpp = use_cpp

    def generate(self, boxes, width, height, chipsize):
        b = np.array(boxes, dtype=np.float64).reshape(-1, 4)
        b[:, 0::2] = np.maximum(np.minimum(b[:, 0::2], width - 2), 0)
        b[:, 1::2] = np.maximum(np.minimum(b[:, 1::2], height - 2), 0)
        return host.chips_generate(b.astype(np.float32), width, height, chipsize, self.chip_stride).tolist()


class chip_worker(object):
    def __init__(self, cfg, chip_size, rng=None):
        """rng: a np.random.RandomState the chip stride is drawn from (default: the global np.random, as the
        reference)."""
        self.valid_ranges = cfg.TRAIN.VALID_RANGES
        self.scales = cfg.TRAIN.SCALES
        self.chip_size = chip_size
        self.use_cpp = cfg.TRAIN.CPP_CHIPS
        self.use_neg_chips = cfg.TRAIN.USE_NEG_CHIPS
        self.rng = rng
        self.reset()

    def reset(self):
        """A new chip stride per epoch (data_workers.py:380, 390-392)."""
        self.chip_stride = (np.random if self.rng is None else self.rng).randint(56, 60)
        self.chip_generator = chip_generator(chip_stride=self.chip_stride, use_cpp=self.use_cpp)

    # ---- helpers
    def _int_sizes(self, boxes):
        w = (boxes[:, 2] - boxes[:, 0]).astype(np.int32)
        h = (boxes[:, 3] - boxes[:, 1]).astype(np.int32)
        return w, h, np.sqrt(w * h), np.maximum(w, h)

    def _fits(self, longest, scale):
        return longest < (self.chip_size - self.chip_stride - 1) / scale

    def _tag(self, chip, scale, idx, r):
        last = idx == len(self.scales) - 1
        if last:      # chips of the coarsest scale carry the resized image size
            return [chip, scale, int(r['height'] * scale), int(r['width'] * scale), idx]
        return [chip, scale, self.chip_size, self.chip_size, idx]

    # ---- positive chips (data_workers.py:394-450)
    def chip_extractor(self, r):
        gt = r['boxes'][np.where(r['max_overlaps'] == 1)[0], :]
        w, h, size, longest = self._int_sizes(gt)
        n = len(self.scales)
        crops = []
        for i, f in enumerate(image_scales(self.scales, r['width'], r['height'])):
            lo, hi = self.valid_ranges[i][0], self.valid_ranges[i][1]
            if i == n - 1:
                sel = size >= lo
            elif i == 0:
                sel = (size < hi) & self._fits(longest, f) & (w >= 2) & (h >= 2)
            else:
                sel = (size >= lo) & (size < hi) & self._fits(longest, f)
            found = self.chip_generator.generate(gt[np.where(sel)[0], :] * f, int(r['width'] * f), int(r['height'] * f),
                                                 self.chip_size)
            for chip in np.array(found) / f:
                crops.append(self._tag(chip, f, i, r))
        return crops

    # ---- box -> chip assignment (+ negative chips) (data_workers.py:452-594)
    def _assign(self, chips, boxes, box_ids, idx, strict_hi):
        """For every box the chip containing most of it (first maximum); the box is kept by that chip iff their
        intersection is at least 1 px on both sides and its sqrt-area is inside the scale's range.  Returns
        (per-chip lists of box ids in box order, kept mask)."""
        per_chip = [[] for _ in range(chips.shape[0])]
        kept = np.zeros(boxes.shape[0], dtype=bool)
        if chips.shape[0] == 0 or boxes.shape[0] == 0:
            return per_chip, kept
        owner = host.ignore_overlaps(chips, boxes).argmax(axis=0)
        c = chips[owner]
        x1, x2 = np.maximum(c[:, 0], boxes[:, 0]), np.minimum(c[:, 2], boxes[:, 2])
        y1, y2 = np.maximum(c[:, 1], boxes[:, 1]), np.minimum(c[:, 3], boxes[:, 3])
        side = np.sqrt(np.abs((x2 - x1) * (y2 - y1)))
        if idx == len(self.scales) - 1:
            in_range = side >= self.valid_ranges[idx][0]
        elif strict_hi:
            in_range = side < self.valid_ranges[idx][1]
        else:
            in_range = side <= self.valid_ranges[idx][1]
        kept = (x2 - x1 >= 1) & (y2 - y1 >= 1) & in_range
        for pi in np.where(kept)[0]:
            per_chip[owner[pi]].append(box_ids[pi])
        return per_chip, kept

    def box_assigner(self, r):
        n = len(self.scales)
        factors = image_scales(self.scales, r['width'], r['height'])
        w, h, size, longest = self._int_sizes(r['boxes'])
        # chips of this image grouped by scale, remembering their position in r['crops']
        by_scale = [[] for _ in range(n)]
        pos = [[] for _ in range(n)]
        for ci, crop in enumerate(r['crops']):
            by_scale[crop[4]].append(crop[0])
            pos[crop[4]].append(ci)
        by_scale = [np.array(c) for c in by_scale]
        # boxes (GT and proposals alike) that a scale is responsible for
        ids = []
        for i, f in enumerate(factors):
            if i == n - 1:
                ids.append(np.where(size >= self.valid_ranges[i][0])[0])
            else:
                ids.append(np.where((size < self.valid_ranges[i][1]) & self._fits(longest, f) & (w >= 2) & (h >= 2))[0])
        boxes = [r['boxes'][k].astype(float) for k in ids]
        props_in_chips = [[] for _ in range(len(r['crops']))]
        covered = []
        for i in range(n):
            per_chip, kept = self._assign(by_scale[i], boxes[i], ids[i], i, strict_hi=False)
            for local, lst in enumerate(per_chip):
                props_in_chips[pos[i][local]] = lst
            covered.append(kept)
        props_in_chips = [np.array(p, dtype=np.int32) for p in props_in_chips]
        if not self.use_neg_chips:
            return [props_in_chips]
        # negative chips: cover what no positive chip kept, keep the crowded ones
        left = [boxes[i][np.where(covered[i] == False)[0]] for i in range(n)]          # noqa: E712
        left_ids = [ids[i][np.where(covered[i] == False)[0]] for i in range(n)]        # noqa: E712
        neg = []
        for i, f in enumerate(factors):
            found = self.chip_generator.generate(left[i] * f, int(r['width'] * f), int(r['height'] * f), self.chip_size)
            neg.append(np.array(found, dtype=float) / f)
        final_chips, final_props = [], []
        for i, f in enumerate(factors):
            per_chip, _ = self._assign(neg[i], left[i], left_ids[i], i, strict_hi=True)
            for chip, lst in zip(neg[i], per_chip):
                if len(lst) > 25 or (len(lst) > 10 and i != 0):
                    final_props.append(np.array(lst, dtype=int))
                    final_chips.append(self._tag(chip, f, i, r))
        r['neg_chips'] = final_chips
        r['neg_props_in_chips'] = final_props
        return props_in_chips, final_chips, final_props
