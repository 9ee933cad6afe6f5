"""AutoFocus inference chips: FocusPixel map -> FocusChips of the next scale, and pruning of chip-border detections.

Host-side mirror of `lib/chips/chips_inference.py` (`gmask` :12-89, `add_chips` :91-173) and of the projection /
`check_valid` step of `Tester.get_detections` (lib/inference.py:235-256, 335-351).  Same function names, argument meaning
and return values as the reference.

The reference leans on OpenCV for three primitives (this image has no OpenCV, so parity of those three is UNPINNED and
restated here from the OpenCV documentation):
  * `cv2.dilate(mask, ones((d, d)))`: max over the d x d window anchored at (d // 2, d // 2), pixels outside ignored;
  * `cv2.findContours(mask, RETR_LIST, ...)`: every outer border (one per 8-connected foreground component) AND every hole
    border (one per background region enclosed by foreground; a hole border runs over the foreground pixels around it);
  * `cv2.boundingRect(contour)`: tight box of the border pixels = the component's box for an outer border, the hole's box
    grown by one pixel for a hole border.
Contours are listed last-found-first (raster scan of the start pixel, the order `RETR_LIST` yields).  Everything else --
the integer arithmetic of the merge loop (Python 2 `/` on ints = floor division), the iteration until the chip count
stops changing, the rescaling -- follows the reference line by line.

The device detection backend leaves its FocusPixel maps on the GPU (`DeviceFocusMaps`); `add_chips` given those runs
`gmask` for every map of the scale in one `ops.focus_chips` launch (csrc/focus_chips.cu), byte-equal to the host code
here, which stays the specification the kernel is tested against.
"""
import math

import numpy as np
from scipy import ndimage

from . import ops

_S8 = np.ones((3, 3), dtype=bool)
_S4 = np.array([[0, 1, 0], [1, 1, 1], [0, 1, 0]], dtype=bool)


def dilate(mask, d):
    """cv2.dilate(mask, np.ones((d, d), np.uint8)) for a 2-D array: dst(y, x) = max src(y + j - a, x + i - a),
    0 <= i, j < d, a = d // 2, positions outside the image skipped."""
    H, W = mask.shape
    a = d // 2
    out = mask.copy()
    for j in range(d):
        for i in range(d):
            dy, dx = j - a, i - a
            ys0, ys1 = max(0, dy), min(H, H + dy)
            xs0, xs1 = max(0, dx), min(W, W + dx)
            if ys0 >= ys1 or xs0 >= xs1:
                continue
            out[ys0 - dy:ys1 - dy, xs0 - dx:xs1 - dx] = np.maximum(out[ys0 - dy:ys1 - dy, xs0 - dx:xs1 - dx],
                                                                   mask[ys0:ys1, xs0:xs1])
    return out


def contour_rects(mask):
    """Bounding rectangles (x, y, w, h) of the borders `cv2.findContours(mask, cv2.RETR_LIST, ...)` returns."""
    fg = mask != 0
    H, W = fg.shape
    found = []                                   # (start_y, start_x, rect)
    lab, n = ndimage.label(fg, structure=_S8)
    for k, sl in enumerate(ndimage.find_objects(lab)):
        ys, xs = sl
        row = np.where(lab[ys.start, xs] == k + 1)[0]
        found.append((ys.start, xs.start + int(row[0]), (xs.start, ys.start, xs.stop - xs.start, ys.stop - ys.start)))
    blab, bn = ndimage.label(~fg, structure=_S4)
    if bn:
        border = set(np.unique(np.concatenate([blab[0, :], blab[-1, :], blab[:, 0], blab[:, -1]])).tolist())
        for k, sl in enumerate(ndimage.find_objects(blab)):
            if (k + 1) in border:
                continue                          # connected to the frame: not a hole
            ys, xs = sl
            x0, y0 = max(xs.start - 1, 0), max(ys.start - 1, 0)
            x1, y1 = min(xs.stop + 1, W), min(ys.stop + 1, H)
            # the border of a hole starts at the foreground pixel left of the hole's first pixel in scan order
            row = np.where(blab[ys.start, xs] == k + 1)[0]
            found.append((ys.start, xs.start + int(row[0]) - 1, (x0, y0, x1 - x0, y1 - y0)))
    found.sort(key=lambda t: (t[0], t[1]), reverse=True)
    return [r for _, _, r in found]


def _place(x, y, w, h, ms, iw, ih):
    """One contour rectangle -> chip rectangle of at least ms x ms cells kept inside the iw x ih map (gmask :30-48)."""
    cx = (x + x + w) // 2
    cy = (y + y + h) // 2
    w = max(ms, w)
    h = max(ms, h)
    if cx + w // 2 >= iw:
        x = iw - w if iw - w >= 0 else 0
    elif cx - w // 2 < 0:
        x = 0
    else:
        x = cx - w // 2
    if cy + h // 2 >= ih:
        y = ih - h if ih - h >= 0 else 0
    elif cy - h // 2 < 0:
        y = 0
    else:
        y = cy - h // 2
    return x, y, w, h


def gmask(mask, d, thresh_value=0.5, ms=16, im_width=0, im_height=0, cscale=1):
    """FocusPixel probability map (stride 16) -> list of FocusChips [x1, y1, x2, y2] in the coordinates of the
    original image (chips_inference.py:12-89)."""
    mask = np.array(mask, copy=True)
    iw = int(math.ceil(float(im_width) / 16))
    ih = int(math.ceil(float(im_height) / 16))
    hi = mask >= thresh_value
    mask[hi] = 1
    mask[~hi] = 0
    mask = dilate(mask, d)
    mask *= 255
    rects = contour_rects(mask.astype(np.uint8))
    chips = []
    nchips = -1
    while nchips != len(chips):
        nchips = len(chips)
        chips = []
        for (x, y, w, h) in rects:
            x, y, w, h = _place(x, y, w, h, ms, iw, ih)
            mask[y:y + h, x:x + w] = 255
        rects = contour_rects(mask.astype(np.uint8))
        for (x, y, w, h) in rects:
            x, y, w, h = _place(x, y, w, h, ms, iw, ih)
            chips.append([x, y, x + w, y + h])
    schips = []
    for c in chips:
        x1, y1, x2, y2 = c[0] * 16, c[1] * 16, c[2] * 16, c[3] * 16
        if x2 > im_width:
            x2 = im_width
            x1 = max(min(x1, x2 - ms * 16), 0)
        if y2 > im_height:
            y2 = im_height
            y1 = max(min(y1, y2 - ms * 16), 0)
        schips.append([x1 / cscale, y1 / cscale, x2 / cscale, y2 / cscale])
    return schips


def image_scale(width, height, target):
    """The resize factor the test iterator applies for TEST.SCALES entry `target` = (min side, max side)."""
    im_size_min, im_size_max = min(width, height), max(width, height)
    s = float(target[0]) / float(im_size_min)
    if np.round(s * im_size_max) > target[1]:
        s = float(target[1]) / float(im_size_max)
    return s


def add_chips(roidb, maps, scale_id, cfg):
    """Replaces every image's `inference_crops` by the FocusChips found at scale `scale_id` (to be processed at scale
    scale_id + 1).  maps[i][j] = (anything, FocusPixel map of crop j of image i).  Returns [chip_area, total_area] in
    megapixels at the next scale (chips_inference.py:91-173).  `maps` may be a `DeviceFocusMaps`: the FocusChips then
    come from the device, with the same values, order and return value."""
    if isinstance(maps, DeviceFocusMaps):
        return _add_chips_device(roidb, maps, scale_id, cfg)
    total_area = 0
    chip_area = 0
    hp = cfg.TEST.CHIP_HYPERPARAMS[scale_id]
    for i, r in enumerate(roidb):
        cur_chips = []
        im_width, im_height = r['width'], r['height']
        cscale = image_scale(im_width, im_height, cfg.TEST.SCALES[scale_id])
        tcscale = image_scale(im_width, im_height, cfg.TEST.SCALES[scale_id + 1])
        total_area = total_area + (im_width * im_height * tcscale * tcscale) / (1000. * 1000.)
        for j in range(len(maps[i])):
            cmap = maps[i][j][1]
            cur_crop = r['inference_crops'][j]
            crop_width = cur_crop[2] - cur_crop[0]
            crop_height = cur_crop[3] - cur_crop[1]
            chips = gmask(cmap, hp[0], hp[1], ms=hp[2], im_width=crop_width * cscale, im_height=crop_height * cscale,
                          cscale=cscale)
            for c in chips:
                c[0] += cur_crop[0]
                c[1] += cur_crop[1]
                c[2] += cur_crop[0]
                c[3] += cur_crop[1]
            for c in chips:
                tarea = (c[2] - c[0]) * (c[3] - c[1]) * tcscale * tcscale
                chip_area = chip_area + tarea / (1000. * 1000.)
            cur_chips += chips
        roidb[i]['inference_crops'] = np.array(cur_chips)
    return [chip_area, total_area]


class DeviceFocusMaps(object):
    """The FocusPixel maps of one test scale as the network left them on the device: per batch the `focus_map` output
    [B, Hc, Wc] (kept alive, not copied) and each row's map extents, ceil(resized h / stride) x ceil(resized w / stride)
    as `Tester._chip_maps` cuts them.  maps[i][j] is (None, host float32 copy of crop j's map of image i), made on
    access, or [] when no batch carried that crop, like the host backend's all_maps; a later batch replaces the map an
    earlier one gave a crop (the iterator repeats crops to fill its batches)."""

    def __init__(self, n_chips, feat_stride):
        self.stride = float(feat_stride)
        self.tensors, self.extents = [], []
        self.where = [[None] * int(n) for n in n_chips]

    def add(self, fm, im_info, im_ids, chip_ids):
        """One batch: fm [B, Hc, Wc] float32 on the device, im_info host float32 [B, 3] (resized h, resized w, scale);
        row b is crop chip_ids[b] of image im_ids[b]."""
        info = np.asarray(im_info, dtype=np.float32).reshape(-1, 3)
        k = len(self.tensors)
        self.tensors.append(fm)
        self.extents.append(np.stack([np.ceil(info[:, 0] / self.stride), np.ceil(info[:, 1] / self.stride)],
                                     1).astype(np.int64))
        for b, (i, j) in enumerate(zip(im_ids, chip_ids)):
            self.where[int(i)][int(j)] = (k, b)

    def __len__(self):
        return len(self.where)

    def __getitem__(self, i):
        return _ImageFocusMaps(self, i)

    def focus_table(self, roidb, scale):
        """The `ops.focus_chips` inputs of every (image, crop) in roidb order: (index int64 [n, 6] = batch, row, H, W,
        iw, ih; geometry float64 [n, 5] = im_width, im_height, cscale, crop x1, crop y1), each value from add_chips' /
        gmask's own expression (cscale = image_scale at `scale`, im_width = crop width * cscale, iw = ceil(im_width /
        16))."""
        index, geometry = [np.zeros((0, 6), np.int64)], [np.zeros((0, 5))]
        for i, r in enumerate(roidb):
            crops = np.asarray(r['inference_crops'])
            if len(crops) != len(self.where[i]):
                raise ValueError("DeviceFocusMaps: image %d has %d crops and %d maps" % (i, len(crops), len(self.where[i])))
            if not len(crops):
                continue
            if any(w is None for w in self.where[i]):
                raise ValueError("DeviceFocusMaps: crop %d of image %d has no map" % (self.where[i].index(None), i))
            crops = crops.reshape(-1, 4)
            cscale = image_scale(r['width'], r['height'], scale)
            imw = np.asarray((crops[:, 2] - crops[:, 0]) * cscale, np.float64)
            imh = np.asarray((crops[:, 3] - crops[:, 1]) * cscale, np.float64)
            kb = np.array(self.where[i], np.int64)
            hw = np.array([self.extents[k][b] for k, b in self.where[i]], np.int64)
            index.append(np.column_stack([kb, hw, np.ceil(imw / 16), np.ceil(imh / 16)]).astype(np.int64))
            geometry.append(np.column_stack([imw, imh, np.full(len(crops), cscale), crops[:, 0], crops[:, 1]])
                            .astype(np.float64))
        return np.concatenate(index), np.concatenate(geometry)


class _ImageFocusMaps(object):
    """maps[i] of a `DeviceFocusMaps`: one entry per crop of image i."""

    def __init__(self, maps, i):
        self._maps, self._where = maps, maps.where[i]

    def __len__(self):
        return len(self._where)

    def __getitem__(self, j):
        w = self._where[j]
        if w is None:
            return []
        k, b = w
        H, W = self._maps.extents[k][b]
        return (None, np.ascontiguousarray(self._maps.tensors[k][b, :H, :W].cpu().numpy()))


def _add_chips_device(roidb, maps, scale_id, cfg):
    """add_chips for a `DeviceFocusMaps`: the FocusChips of every map from one `ops.focus_chips` launch, then the area
    sums on the host with add_chips' expressions, in its order."""
    hp = cfg.TEST.CHIP_HYPERPARAMS[scale_id]
    index, geometry = maps.focus_table(roidb, cfg.TEST.SCALES[scale_id])
    chips, off = ops.focus_chips(maps.tensors, index, geometry, d=hp[0], thresh=hp[1], ms=hp[2])
    total_area = 0
    chip_area = 0
    m = 0
    for i, r in enumerate(roidb):
        im_width, im_height = r['width'], r['height']
        tcscale = image_scale(im_width, im_height, cfg.TEST.SCALES[scale_id + 1])
        total_area = total_area + (im_width * im_height * tcscale * tcscale) / (1000. * 1000.)
        n = len(maps[i])
        cur = chips[off[m]:off[m + n]]
        m += n
        for c in cur:
            tarea = (c[2] - c[0]) * (c[3] - c[1]) * tcscale * tcscale
            chip_area = chip_area + tarea / (1000. * 1000.)
        roidb[i]['inference_crops'] = cur.copy() if len(cur) else np.array([])
    return [chip_area, total_area]


def check_valid(det, chip, im_width, im_height, delta=10):
    """A detection within `delta` px of a chip border that is not an image border is cut off by the chip: drop it
    (Tester.get_detections, lib/inference.py:235-256)."""
    dx1, dy1, dx2, dy2 = det[0], det[1], det[2], det[3]
    cx1, cy1, cx2, cy2 = chip[0], chip[1], chip[2], chip[3]
    if cx1 >= 0.5 and abs(dx1 - cx1) < delta:
        return False
    if cy1 >= 0.5 and abs(dy1 - cy1) < delta:
        return False
    if cx2 < im_width - 0.5 and abs(dx2 - cx2) < delta:
        return False
    if cy2 < im_height - 0.5 and abs(dy2 - cy2) < delta:
        return False
    return True


def prune_mask(d, chip, im_width, im_height, delta=10):
    """check_valid for every row of d ([n, >=4], image coordinates) at once."""
    keep = np.ones(d.shape[0], dtype=bool)
    if chip[0] >= 0.5:
        keep &= ~(np.abs(d[:, 0] - chip[0]) < delta)
    if chip[1] >= 0.5:
        keep &= ~(np.abs(d[:, 1] - chip[1]) < delta)
    if chip[2] < im_width - 0.5:
        keep &= ~(np.abs(d[:, 2] - chip[2]) < delta)
    if chip[3] < im_height - 0.5:
        keep &= ~(np.abs(d[:, 3] - chip[3]) < delta)
    return keep


def project_and_prune(cls_dets, chip, im_width, im_height, delta=10):
    """Detections of one chip (chip coordinates, rows x1 y1 x2 y2 score) -> image coordinates, border-cut ones removed
    (`do_pruning` branch, lib/inference.py:335-351).  Vectorised form of the per-detection loop."""
    d = np.array(cls_dets, dtype=np.float64, copy=True).reshape(-1, 5)
    if d.shape[0] == 0:
        return np.zeros((0, 5))
    d[:, 0] += chip[0]; d[:, 2] += chip[0]
    d[:, 1] += chip[1]; d[:, 3] += chip[1]
    d = d[prune_mask(d, chip, im_width, im_height, delta)]
    return d if d.shape[0] > 0 else np.zeros((0, 5))
