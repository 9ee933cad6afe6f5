"""The SNIPER training iterator with a GPU input stage.

Host side (`MNIteratorE2E`): same construction arguments, epoch logic and per-chip bookkeeping as the reference's
lib/iterators/MNIteratorE2E.py -- `reset()` (:41-105: chip extraction, box assignment and negative-chip mining through
`chip_worker`, <= 2 negative chips per image, padding of the chip list to a multiple of the batch, permutation) and
`_get_batch()` (:112-219: chip selection through `chip_order` / `crop_idx`, valid ranges, im_info, the GT bookkeeping in
front of the anchor matching, data_workers.py:194-281) -- but instead of resizing pixels and matching anchors in a
`Pool(64)` of host processes it emits a small pinned **raw batch**: the uint8 source rectangle of every chip, a chip
table, and the (valid GT, invalid GT, gt_boxes) arrays.

Device side (`InputStage`): one H2D copy of that raw batch, then `sniper_chip_input` (flip + cv2-style bilinear resize
+ pad + BGR->RGB + mean subtraction, data_workers.py:80-121), `sniper_anchor_target` (anchor matching, :283-363) and
`sniper_anchor_subsample` (the npr.choice subsampling, :326-338) fill exactly the tensors `MNIteratorE2E.provide_data /
provide_label` name: data, valid_ranges, im_info, label, bbox_target, bbox_weight, gt_boxes (SURVEY appendix B.5).

What stays on the host is what north_star keeps there: lib/chips sampling and the iterator's index logic.

Data parallel (`rank=`): the reference builds ONE iterator over the global batch of nGPUs * BATCH_IMAGES chips and MXNet
hands GPU g the slice [g*B, (g+1)*B) of every batch (executor_manager._split_input_slice).  Here every rank runs its
own iterator over the same roidb with the same `seed`: each computes the whole epoch plan, identically, and builds only
its own slice.  `RawBatch.chip_base` carries the slice's position, so the device subsampling draws what the global
batch would (`sniper_anchor_subsample_at`), and `RawBatch.plan_digest` lets Trainer.fit check that the ranks agree.
"""
import hashlib
import math

import numpy as np
import torch

from . import host, ops
from ._lib import check, lib
from .chip_worker import chip_worker


def _clip(boxes, im_shape):
    """bbox_transform.clip_boxes (lib/bbox/bbox_transform.py:35-50), in place like the reference."""
    boxes[:, 0::4] = np.maximum(np.minimum(boxes[:, 0::4], im_shape[1] - 1), 0)
    boxes[:, 1::4] = np.maximum(np.minimum(boxes[:, 1::4], im_shape[0] - 1), 0)
    boxes[:, 2::4] = np.maximum(np.minimum(boxes[:, 2::4], im_shape[1] - 1), 0)
    boxes[:, 3::4] = np.maximum(np.minimum(boxes[:, 3::4], im_shape[0] - 1), 0)
    return boxes


def _big_enough(boxes, min_size):
    ws = boxes[:, 2] - boxes[:, 0] + 1
    hs = boxes[:, 3] - boxes[:, 1] + 1
    return np.where((ws >= min_size) & (hs >= min_size))[0]


def _to_chip(boxes, im_info, cur_crop, im_scale):
    """shift into the chip (in place), scale, round, clip to the chip (data_workers.py:208-224)"""
    boxes[:, 0] -= cur_crop[0]
    boxes[:, 2] -= cur_crop[0]
    boxes[:, 1] -= cur_crop[1]
    boxes[:, 3] -= cur_crop[1]
    return _clip(np.round(boxes * im_scale), im_info[:2])


def chip_focus_boxes(im_info, cur_crop, im_scale, gt_boxes):
    """The boxes gen_mask reads (data_workers.py:220-222): EVERY GT box of the image shifted into the chip, scaled,
    rounded and clipped to it, before the 10 px filter (a box outside the chip becomes a zero-width box on its border)."""
    return _to_chip(np.array(gt_boxes, copy=True).reshape(-1, 4), im_info, cur_crop, im_scale)


def chip_ground_truth(im_info, cur_crop, im_scale, nids, gtids, gt_boxes, boxes, classes, max_n_gts=100):
    """The GT bookkeeping of anchor_worker.worker in front of the anchor matching (data_workers.py:194-281):
    shift into the chip, scale, round, clip to the chip, drop boxes under 10 px, then split the chip's GT into
    `valid` (GT this chip is responsible for: it coincides with a box of props_in_chips) and `invalid` (other GT that
    fall into the chip: anchors on them are ignored).  Returns (valid [n,4], invalid [m,4], gt_boxes [max_n_gts,5])."""
    gt_boxes = np.array(gt_boxes, copy=True)
    boxes = np.asarray(boxes)
    vgt = boxes[np.intersect1d(gtids, nids)]          # fancy indexing: a copy
    gt_boxes = _to_chip(gt_boxes, im_info, cur_crop, im_scale)
    vgt = _to_chip(vgt, im_info, cur_crop, im_scale)
    ids = _big_enough(gt_boxes, 10)
    if len(ids) == 0:
        gt_boxes = np.zeros((0, 4))
        classes = np.zeros((0, 1))
    else:
        gt_boxes = gt_boxes[ids]
        classes = classes[ids]
    all_gt = gt_boxes.copy()
    ids = _big_enough(vgt, 10)
    vgt = vgt[ids] if len(ids) > 0 else np.zeros((0, 4))
    if len(vgt) > 0 and len(gt_boxes) > 0:
        mov = host.bbox_overlaps(gt_boxes.astype(float), vgt.astype(float)).max(axis=1)
    else:
        mov = np.zeros((len(gt_boxes)))
    invalid = gt_boxes[np.where(mov < 1)[0], :]
    valid = gt_boxes[np.where(mov == 1)[0], :]
    fgt = -np.ones((max_n_gts, 5))
    if len(all_gt) > 0:
        k = min(len(all_gt), max_n_gts)
        fgt[:k, :] = np.hstack((all_gt, classes))[:k]
    return valid, invalid, fgt


class RawBatch(object):
    """Pinned host buffers of one batch (what crosses PCIe): source pixels + small per-chip arrays.

    MNIteratorE2E reuses a ring of `n_buffers` of these.  InputStage.run copies a batch to the device with
    asynchronous H2D copies, so a buffer may be refilled only after the step that read it has completed.  A caller
    that synchronises every step (Trainer.step_raw) needs depth + 2 buffers behind a PrefetchingIter of that depth;
    Trainer.fit keeps the host at most one step ahead (it waits for step i-1 before it takes batch i+1), so two
    batches can be in flight and it needs depth + 3."""

    def __init__(self, B, max_gt, pixel_capacity, focus_cap=0):
        """focus_cap > 0 (TRAIN.AUTO_FOCUS): room for that many FocusPixel boxes per chip (`focus_boxes`, `nfocus`)."""
        can_pin = torch.cuda.is_available()          # host-only use (tests without a GPU): plain pageable buffers

        def pin(*s, dtype):
            t = torch.zeros(*s, dtype=dtype)
            return t.pin_memory() if can_pin else t
        self.focus_boxes = pin(B, focus_cap, 4, dtype=torch.float32) if focus_cap > 0 else None
        self.nfocus = pin(B, dtype=torch.int32) if focus_cap > 0 else None
        self.pixels = pin(pixel_capacity, dtype=torch.uint8)
        self.table = pin(B, 8, dtype=torch.int64)
        self.valid_ranges = pin(B, 2, dtype=torch.float32)
        self.im_info = pin(B, 3, dtype=torch.float32)
        self.gt_valid = pin(B, max_gt, 4, dtype=torch.float32)
        self.ngt = pin(B, dtype=torch.int32)
        self.gt_invalid = pin(B, max_gt, 4, dtype=torch.float32)
        self.ninv = pin(B, dtype=torch.int32)
        self.gt_boxes = pin(B, max_gt, 5, dtype=torch.float32)
        self.anchor_im_info = pin(B, 3, dtype=torch.float32)
        self.used_pixels = 0
        self.seed = 0
        self.chip_base = 0           # position of chip 0 of this batch in the global batch (data parallel: rank * B)
        self.plan_digest = None      # 64-bit digest of the epoch plan the batch comes from (MNIteratorE2E.plan_digest)

    def nbytes(self):
        small = (self.table, self.valid_ranges, self.im_info, self.gt_valid, self.ngt, self.gt_invalid, self.ninv,
                 self.gt_boxes, self.anchor_im_info)
        if self.focus_boxes is not None:
            small += (self.focus_boxes, self.nfocus)
        return int(self.used_pixels + sum(t.numel() * t.element_size() for t in small))


def roidb_digest(roidb):
    """64-bit digest of a training roidb: its size and, per entry, the image path, size, flip and boxes."""
    h = hashlib.blake2b(digest_size=8)
    h.update(np.int64(len(roidb)).tobytes())
    for r in roidb:
        h.update(str(r.get('image', '')).encode())
        h.update(np.array([r['width'], r['height'], bool(r.get('flipped', False))], np.int64).tobytes())
        h.update(np.ascontiguousarray(r['boxes'], np.float64).tobytes())
    return int.from_bytes(h.digest(), 'little')


class MNIteratorE2E(object):
    def __init__(self, roidb, config, batch_size=4, threads=8, nGPUs=1, pad_rois_to=400, crop_size=(512, 512),
                 image_loader=None, n_buffers=3, rank=None, seed=None, plan_backend="host", device=None):
        """roidb entries: 'image' (path) or 'image_data' (decoded uint8 HxWx3 BGR), 'width', 'height', 'boxes' [n,4],
        'max_overlaps' (== 1 for GT rows), 'max_classes', 'flipped'.  image_loader(path) -> uint8 BGR array replaces
        cv2.imread (this image has no OpenCV).

        batch_size is the GLOBAL batch (nGPUs * TRAIN.BATCH_IMAGES, main_train.py:44-45).  rank=None yields whole
        batches; rank=r (data parallel, one iterator per rank) yields batches of B = batch_size // nGPUs chips, chips
        [r*B, (r+1)*B) of the global batch the rank=None iterator with the same seed yields.  Every rank computes the
        whole epoch plan (chips, padding, permutation, chip order), so len() and the epoch length are the global ones.
        seed=int: every draw of an epoch comes from a private np.random.RandomState(seed) -- the chip stride, the
        negative-chip pick, the chip permutation, each image's chip_order -- and each epoch seeds the C rand() stream
        of the chip generator from it; seed=None draws from the global np.random (the reference's behaviour).  rank
        needs a seed: the plan is computed on the prefetch thread, where the global state cannot be shared.
        plan_backend="device" computes each epoch's chips, box assignment and negative chips (chip_worker's
        chip_extractor / box_assigner) on `device` (default: the current CUDA device) with chip_plan.DevicePlan, on its
        own stream; the result, including the rand() stream's position, is the host's.  The stride draw, the rand()
        seeding, the negative-chip pick, the permutation and chip_order stay on the host.  The device plan reads the
        roidb's boxes and sizes once, here."""
        if plan_backend not in ("host", "device"):
            raise ValueError("MNIteratorE2E: plan_backend must be 'host' or 'device', not %r" % (plan_backend,))
        assert batch_size % nGPUs == 0, 'batch_size should be divisible by number of GPUs'
        if rank is not None:
            if seed is None:
                raise ValueError("MNIteratorE2E: rank=%r needs a seed (every rank must draw the same epoch plan)" % rank)
            if not 0 <= rank < nGPUs:
                raise ValueError("MNIteratorE2E: rank %r is not in [0, nGPUs = %d)" % (rank, nGPUs))
        self.roidb = roidb
        self.cfg = config
        self.batch_size = batch_size
        self.nGPUs = nGPUs
        self.rank = rank
        self.slice_size = batch_size if rank is None else batch_size // nGPUs
        self.chip_base = 0 if rank is None else rank * self.slice_size
        self.rng = None if seed is None else np.random.RandomState(seed)
        self._roidb_digest = roidb_digest(roidb)
        self.plan_digest = None
        self.crop_size = crop_size
        self.image_loader = image_loader
        self.pixel_mean = config.network.PIXEL_MEANS
        self.chip_worker = chip_worker(chip_size=self.crop_size[0], cfg=config, rng=self.rng)
        self.plan_backend = plan_backend
        self._device_plan = None
        if plan_backend == "device":
            from .chip_plan import DevicePlan
            self._device_plan = DevicePlan(roidb, self.chip_worker, device)
        self.max_gt = 100
        self.data_name = ['data', 'valid_ranges', 'im_info']
        self.label_name = ['label', 'bbox_target', 'bbox_weight', 'gt_boxes']
        # TRAIN.AUTO_FOCUS: every GT box of a chip's image feeds its FocusPixel label (MNIteratorE2E.py:146-147), so the
        # per-chip box capacity is the largest GT count of the roidb
        self.autofocus = bool(getattr(config.TRAIN, 'AUTO_FOCUS', False))
        self.focus_cap = 0
        if self.autofocus:
            self.label_name.append('scale_label')
            self.focus_cap = max([int((r['max_overlaps'] == 1).sum()) for r in roidb] + [1])
        self.epiter = 0
        # the largest source rectangle of a chip: crop_size / (smallest scale factor) on each side, x3 channels
        self._buffers = [None] * n_buffers
        self._next_buffer = 0
        self.batch = None
        self.reset()

    # ---------------------------------------------------------------- epoch (MNIteratorE2E.py:41-105)
    def reset(self):
        npr = np.random if self.rng is None else self.rng
        self.cur_i = 0
        self.n_neg_per_im = 2
        self.crop_idx = [0] * len(self.roidb)
        self.chip_worker.reset()
        if self.rng is not None:
            host.srand(int(self.rng.randint(0, 2 ** 31)))
        chip_count = 0
        if self._device_plan is not None:
            self._device_plan.plan(self.roidb)
            chip_count = sum(len(r['crops']) for r in self.roidb)
        else:
            for r in self.roidb:
                r['crops'] = self.chip_worker.chip_extractor(r)
                chip_count += len(r['crops'])
            for r in self.roidb:
                ps = self.chip_worker.box_assigner(r)
                r['props_in_chips'] = ps[0]
                if self.cfg.TRAIN.USE_NEG_CHIPS:
                    r['neg_crops'] = ps[1]
                    r['neg_props_in_chips'] = ps[2]
        chipindex = []
        for i, r in enumerate(self.roidb):
            if self.cfg.TRAIN.USE_NEG_CHIPS:
                cs = r['neg_crops']
                if len(cs) > 0:
                    sel_inds = np.arange(len(cs))
                    if len(cs) > self.n_neg_per_im:
                        sel_inds = npr.permutation(sel_inds)[0:self.n_neg_per_im]
                    for ind in sel_inds:
                        chip_count += 1
                        r['crops'].append(r['neg_crops'][ind])
                        r['props_in_chips'].append(r['neg_props_in_chips'][ind].astype(np.int32))
            chipindex += [i] * len(r['crops'])
        self.chip_count = chip_count
        chipindex = np.array(chipindex)
        if chipindex.shape[0] % self.batch_size > 0:
            extra = self.batch_size - (chipindex.shape[0] % self.batch_size)
            chipindex = np.hstack((chipindex, chipindex[0:extra]))
        self.inds = np.array(npr.permutation(chipindex), dtype=int)
        for r in self.roidb:
            r['chip_order'] = npr.permutation(np.arange(len(r['crops'])))
        self.epiter += 1
        self.size = len(self.inds)
        self.plan_digest = self._digest()

    def _digest(self):
        """64-bit digest of this epoch's plan: the roidb (roidb_digest), the chip stride, the chip count, the padded
        chip permutation `inds`, and every image's chips and chip order."""
        h = hashlib.blake2b(digest_size=8)
        h.update(np.array([self._roidb_digest, self.chip_worker.chip_stride, self.chip_count, len(self.inds)],
                          np.uint64).tobytes())
        h.update(np.ascontiguousarray(self.inds, np.int64).tobytes())
        for r in self.roidb:
            h.update(np.array([c[0] for c in r['crops']], np.float64).tobytes())
            h.update(np.ascontiguousarray(r['chip_order'], np.int64).tobytes())
        return int.from_bytes(h.digest(), 'little')

    def __len__(self):
        return len(self.inds)

    def __iter__(self):
        return self

    def __next__(self):
        if not self.get_batch():
            raise StopIteration
        return self.batch

    next = __next__

    def get_batch(self):
        if self.cur_i >= self.size:
            return False
        self.batch = self._get_batch()
        self.cur_i += self.batch_size
        return True

    # ---------------------------------------------------------------- one batch (MNIteratorE2E.py:112-219)
    def _image(self, r):
        if 'image_data' in r:
            return r['image_data']
        if self.image_loader is None:
            raise RuntimeError("roidb entry has no 'image_data' and no image_loader was given (no OpenCV in this image)")
        return self.image_loader(r['image'])

    def _raw(self, need_pixels):
        i = self._next_buffer
        self._next_buffer = (i + 1) % len(self._buffers)
        buf = self._buffers[i]
        if buf is None or buf.pixels.numel() < need_pixels:
            buf = self._buffers[i] = RawBatch(self.slice_size, self.max_gt, int(need_pixels * 1.25) + 4096,
                                              self.focus_cap)
        return buf

    def _get_batch(self):
        cur_from, cur_to = self.cur_i, self.cur_i + self.batch_size
        entries = [self.roidb[self.inds[i]] for i in range(cur_from, cur_to)]
        cropids = [r['chip_order'][self.crop_idx[self.inds[i]] % len(r['chip_order'])]
                   for r, i in zip(entries, range(cur_from, cur_to))]
        for i in range(cur_from, cur_to):
            self.crop_idx[self.inds[i]] += 1
        # data parallel: the crop_idx of every chip of the global batch has moved on; this rank builds only its slice
        mine = slice(self.chip_base, self.chip_base + self.slice_size)
        entries, cropids = entries[mine], cropids[mine]
        # source rectangles (im_worker.worker: flip, then im[int(y1):int(y2), int(x1):int(x2)])
        rects = []
        for r, cid in zip(entries, cropids):
            crop = r['crops'][cid]
            im = self._image(r)
            H, W = im.shape[0], im.shape[1]
            x1, y1, x2, y2 = int(crop[0][0]), int(crop[0][1]), int(crop[0][2]), int(crop[0][3])
            y1c, y2c = min(max(y1, 0), H), min(max(y2, 0), H)
            x1c, x2c = min(max(x1, 0), W), min(max(x2, 0), W)
            if r.get('flipped', False):      # columns [x1, x2) of the flipped image = [W - x2, W - x1) of the stored one
                xa, xb = W - x2c, W - x1c
            else:
                xa, xb = x1c, x2c
            rects.append((im, y1c, y2c, xa, xb))
        need = sum(max(y2 - y1, 0) * max(xb - xa, 0) * 3 for _, y1, y2, xa, xb in rects)
        raw = self._raw(need)
        pix = raw.pixels.numpy()
        off = 0
        S0, S1 = self.crop_size
        for k, (r, cid, (im, y1, y2, xa, xb)) in enumerate(zip(entries, cropids, rects)):
            crop = r['crops'][cid]
            im_scale = crop[1]
            h, w = max(y2 - y1, 0), max(xb - xa, 0)
            n = h * w * 3
            if n:
                pix[off:off + n].reshape(h, w, 3)[...] = im[y1:y2, xa:xb, :3]
            dst_h, dst_w = int(np.rint(h * im_scale)), int(np.rint(w * im_scale))      # cv2.resize dsize = cvRound(...)
            raw.table[k] = torch.tensor([off, h, w, dst_h, dst_w, 1 if r.get('flipped', False) else 0,
                                         int(np.float64(im_scale).view(np.int64)), 0], dtype=torch.int64)
            off += n
            scalei, height, width = crop[4], crop[2], crop[3]
            vr = self.cfg.TRAIN.VALID_RANGES[scalei]
            raw.valid_ranges[k, 0] = 0 if vr[0] < 0 else vr[0] * im_scale
            raw.valid_ranges[k, 1] = S1 if vr[1] < 0 else vr[1] * im_scale
            raw.im_info[k] = torch.tensor([height, width, im_scale], dtype=torch.float32)
            # the anchor matcher sees the chip as a full crop_size x crop_size image (MNIteratorE2E.py:137)
            info = [S0, S1, im_scale]
            raw.anchor_im_info[k] = torch.tensor(info, dtype=torch.float32)
            gtids = np.where(r['max_overlaps'] == 1)[0]
            classes = r['max_classes'][gtids]
            valid, invalid, fgt = chip_ground_truth(info, crop[0], im_scale, r['props_in_chips'][cid], gtids,
                                                    r['boxes'][gtids, :], r['boxes'].copy(),
                                                    classes.reshape(len(classes), 1), self.max_gt)
            nv, ni = min(len(valid), self.max_gt), min(len(invalid), self.max_gt)
            raw.ngt[k], raw.ninv[k] = nv, ni
            if nv:
                raw.gt_valid[k, :nv] = torch.from_numpy(np.ascontiguousarray(valid[:nv], dtype=np.float32))
            if ni:
                raw.gt_invalid[k, :ni] = torch.from_numpy(np.ascontiguousarray(invalid[:ni], dtype=np.float32))
            raw.gt_boxes[k] = torch.from_numpy(fgt.astype(np.float32))
            if self.autofocus:
                fb = chip_focus_boxes(info, crop[0], im_scale, r['boxes'][gtids, :])
                if len(fb) > raw.focus_boxes.shape[1]:
                    raise ValueError("chip has %d GT boxes, more than the FocusPixel capacity %d (the roidb changed "
                                     "after the iterator was built)" % (len(fb), raw.focus_boxes.shape[1]))
                raw.nfocus[k] = len(fb)
                if len(fb):
                    raw.focus_boxes[k, :len(fb)] = torch.from_numpy(np.ascontiguousarray(fb, dtype=np.float32))
        raw.used_pixels = off
        raw.seed = (self.epiter * 1000003 + self.cur_i) & 0x7FFFFFFF
        raw.chip_base = self.chip_base
        raw.plan_digest = self.plan_digest
        return raw


EPOCH_END = object()      # what PrefetchingIter(epoch_marker=True) yields after the last batch of every epoch


class PrefetchingIter(object):
    """Background-thread prefetch of raw batches (the role of mx.io.PrefetchingIter around MNIteratorE2E in
    main_train.py): the host bookkeeping of batch i+1 runs while the GPU computes batch i.  The wrapped iterator must
    own at least depth + 2 raw buffers (n_buffers; depth + 3 under Trainer.fit, see RawBatch).  Epochs follow each
    other silently unless epoch_marker=True, which yields `EPOCH_END` after each one."""

    def __init__(self, it, depth=2, epochs=None, epoch_marker=False):
        import queue
        import threading
        self.it = it
        self.q = queue.Queue(maxsize=depth)
        self.epochs = epochs
        self.epoch_marker = epoch_marker
        self._stop = False
        # Every ctypes call of the training step releases the GIL and has to win it back from the producer thread; with
        # the default 5 ms switch interval each of those hand-overs can stall the step by up to 5 ms (measured: step_raw
        # 56 ms instead of 36 ms next to a busy producer).  0.5 ms keeps the hand-over cost small.
        import sys
        self._switch = sys.getswitchinterval()
        sys.setswitchinterval(5e-4)
        self.th = threading.Thread(target=self._run, daemon=True)
        self.th.start()

    def _run(self):
        ep = 0
        while not self._stop:
            for raw in self.it:
                if self._stop:
                    return
                self.q.put(raw)
            if self.epoch_marker:
                self.q.put(EPOCH_END)
            ep += 1
            if self.epochs is not None and ep >= self.epochs:
                self.q.put(None)
                return
            self.it.reset()

    def __iter__(self):
        return self

    def __next__(self):
        raw = self.q.get()
        if raw is None:
            raise StopIteration
        return raw

    def close(self):
        """Stops and JOINS the worker (a daemon thread still inside a ctypes call when the interpreter exits aborts the
        process): keep draining the queue so that a worker blocked in put() can see the stop flag."""
        import queue
        self._stop = True
        while self.th.is_alive():
            try:
                while True:
                    self.q.get_nowait()
            except queue.Empty:
                pass
            self.th.join(timeout=0.02)
        import sys
        sys.setswitchinterval(self._switch)


class InputStage(object):
    """Device half of the iterator: raw batch -> the network's input tensors (all on `device`)."""

    def __init__(self, cfg, device, batch_size, crop_size=512, max_gt=100):
        self.cfg = cfg
        self.device = torch.device(device)
        self.B, self.S, self.max_gt = batch_size, crop_size, max_gt
        net = cfg.network
        self.scales, self.ratios, self.stride = tuple(net.ANCHOR_SCALES), tuple(net.ANCHOR_RATIOS), net.RPN_FEAT_STRIDE
        self.rpn_batch = cfg.TRAIN.RPN_BATCH_SIZE
        self.num_fg = int(self.rpn_batch * cfg.TRAIN.RPN_FG_FRACTION)
        self.pos, self.neg = cfg.TRAIN.RPN_POSITIVE_OVERLAP, cfg.TRAIN.RPN_NEGATIVE_OVERLAP
        self.means = torch.tensor(list(net.PIXEL_MEANS), dtype=torch.float32, device=self.device)
        self.pixels = None
        z = lambda *s, dtype=torch.float32: torch.zeros(*s, dtype=dtype, device=self.device)
        B = batch_size
        self.dev = dict(table=z(B, 8, dtype=torch.int64), valid_ranges=z(B, 2), im_info=z(B, 3), gt_valid=z(B, max_gt, 4),
                        ngt=z(B, dtype=torch.int32), gt_invalid=z(B, max_gt, 4), ninv=z(B, dtype=torch.int32),
                        gt_boxes=z(B, max_gt, 5), anchor_im_info=z(B, 3))
        self.data = z(B, 3, crop_size, crop_size)
        tr = cfg.TRAIN
        self.autofocus = bool(getattr(tr, 'AUTO_FOCUS', False))
        if self.autofocus:
            self.focus_thresh = (tr.AUTO_FOCUS_DC_LOW, tr.AUTO_FOCUS_SMALL_THRESH, tr.AUTO_FOCUS_DC_HIGH)
            Hf = crop_size // self.stride
            self.scale_label = z(B, Hf * Hf)
            self.focus_dev = None           # [B, cap, 4] device copy of the raw batch's boxes (sized by the first batch)
            self.nfocus = z(B, dtype=torch.int32)

    def run(self, raw, subsample=True):
        """H2D of the raw batch + the three kernels; returns the batch dict Trainer / SniperResNet101 consume.  Everything
        is enqueued on the current stream; the returned tensors are owned by this object and overwritten by the next
        call."""
        n = raw.used_pixels
        if self.pixels is None or self.pixels.numel() < n:
            self.pixels = torch.empty(int(n * 1.25) + 4096, dtype=torch.uint8, device=self.device)
        self.pixels[:n].copy_(raw.pixels[:n], non_blocking=True)
        for k in self.dev:
            self.dev[k].copy_(getattr(raw, k), non_blocking=True)
        st = torch.cuda.current_stream().cuda_stream
        check(lib().sniper_chip_input(self.pixels.data_ptr(), self.dev["table"].data_ptr(), self.means.data_ptr(),
                                      self.data.data_ptr(), self.B, self.S, st))
        Hf = self.S // self.stride
        label, bt, bw = ops.anchor_target(self.dev["gt_valid"], self.dev["ngt"], self.dev["gt_invalid"], self.dev["ninv"],
                                          self.dev["anchor_im_info"], H=Hf, W=Hf, feat_stride=self.stride,
                                          scales=self.scales, ratios=self.ratios, pos_thresh=self.pos,
                                          neg_thresh=self.neg)
        if subsample:
            # keyed by the chip's position in the global batch: a data-parallel rank draws what the whole batch would
            A = len(self.scales) * len(self.ratios)
            check(lib().sniper_anchor_subsample_at(label.data_ptr(), bt.data_ptr(), bw.data_ptr(), self.B, A, Hf, Hf,
                                                   self.num_fg, self.rpn_batch, int(raw.seed), int(raw.chip_base), st))
        out = dict(data=self.data, label=label, bbox_target=bt, bbox_weight=bw, gt_boxes=self.dev["gt_boxes"],
                   valid_ranges=self.dev["valid_ranges"], im_info=self.dev["im_info"])
        if self.autofocus:
            if raw.focus_boxes is None:
                raise ValueError("InputStage: TRAIN.AUTO_FOCUS is set but the raw batch carries no FocusPixel boxes")
            if self.focus_dev is None or self.focus_dev.shape != raw.focus_boxes.shape:
                self.focus_dev = torch.empty(raw.focus_boxes.shape, device=self.device)
            self.focus_dev.copy_(raw.focus_boxes, non_blocking=True)
            self.nfocus.copy_(raw.nfocus, non_blocking=True)
            lo, small, hi = self.focus_thresh
            out["scale_label"] = ops.focus_label(self.focus_dev, self.nfocus, H=Hf, W=Hf, feat_stride=self.stride,
                                                 dc_low=lo, small_thresh=small, dc_high=hi, out=self.scale_label)
        return out


def synthetic_roidb(n_images, seed=0, width=1333, height=800, n_gt=(1, 20), n_prop=300, num_classes=81):
    """COCO-shaped synthetic roidb with decoded images in memory (no dataset, no OpenCV in this image): random uint8
    pixels, GT boxes with sqrt(area) log-uniform in [8, 400] px (SURVEY 8d), a few hundred proposals, random flips."""
    rng = np.random.RandomState(seed)
    out = []
    for i in range(n_images):
        W, H = (width, height) if rng.rand() < 0.7 else (height, width)
        g = int(rng.randint(n_gt[0], n_gt[1] + 1))
        n = g + n_prop
        s = np.exp(rng.uniform(np.log(8), np.log(400), n))
        ar = np.exp(rng.uniform(np.log(0.5), np.log(2.0), n))
        w, h = s * np.sqrt(ar), s / np.sqrt(ar)
        cx, cy = rng.uniform(0, W, n), rng.uniform(0, H, n)
        boxes = np.stack([np.clip(cx - w / 2, 0, W - 1), np.clip(cy - h / 2, 0, H - 1),
                          np.clip(cx + w / 2, 0, W - 1), np.clip(cy + h / 2, 0, H - 1)], 1).astype(np.float32)
        out.append({'image_data': rng.randint(0, 256, (H, W, 3)).astype(np.uint8), 'width': W, 'height': H,
                    'boxes': boxes, 'flipped': bool(rng.rand() < 0.5),
                    'max_overlaps': np.concatenate([np.ones(g), rng.uniform(0, 0.9, n_prop)]).astype(np.float32),
                    'max_classes': np.concatenate([rng.randint(1, num_classes, g), np.zeros(n_prop)]).astype(np.int32)})
    return out


def default_config(neg=True, autofocus=False, network="resnet101", dataset="coco"):
    """The slice of configs/faster/sniper_res101_e2e.yml the iterator reads (:21-39, 76-101, 120-140); autofocus=True:
    TRAIN.AUTO_FOCUS of configs/faster/sniper_res101_e2e_autofocus.yml (FocusPixel labels, thresholds 5 / 64 / 90).
    network="mobilenetv2": the network and TEST blocks of configs/faster/sniper_mobilenetv2_e2e.yml instead (stride 32,
    scales 1 / 2 / 4 / 8 / 12: 15 anchors; plain multi-scale inference without AutoFocus), for
    model_mnv2.SniperMobileNetV2.
    dataset="pascal_voc" (network "resnet101"): the blocks of configs/faster/sniper_res101_e2e_pascal_voc.yml instead,
    for a 21-class SniperResNet101 evaluated by pascal_voc.PascalVOC; its TRAIN block is the COCO yml's.
    The roidb keys of load_data (TRAIN.FLIP, the FG / BG thresholds, TRAIN.BBOX_*, CLASS_AGNOSTIC and dataset.dataset,
    the name load_data.load_proposal_roidb takes) have the same values in every shipped yml (:11, :116-172)."""
    import types
    S = types.SimpleNamespace
    if network == "resnet101":
        net = S(PIXEL_MEANS=[103.06, 115.90, 123.15], ANCHOR_SCALES=[2, 4, 7, 10, 13, 16, 24], ANCHOR_RATIOS=[0.5, 1, 2],
                RPN_FEAT_STRIDE=16, NUM_ANCHORS=21)
        # TEST block of configs/faster/sniper_res101_e2e_autofocus.yml:191-245 (AutoFocus inference, BASELINE config 5)
        test = S(SCALES=[(480, 512), (800, 1280), (1400, 2000)], BATCH_IMAGES=[8, 8, 2], MAX_PER_IMAGE=200,
                 VALID_RANGES=[(75, -1), (32, 180), (-1, 75)], AUTO_FOCUS=True, DO_PRUNING=[False, True, True],
                 CHIP_HYPERPARAMS=[(3, 0.02, 16), (3, 0.2, 20)], NMS=0.45, NMS_SIGMA=0.55)
    elif network == "mobilenetv2":
        net = S(PIXEL_MEANS=[103.939, 116.779, 123.68], ANCHOR_SCALES=[1, 2, 4, 8, 12], ANCHOR_RATIOS=[0.5, 1, 2],
                RPN_FEAT_STRIDE=32, NUM_ANCHORS=15)
        # TEST block of configs/faster/sniper_mobilenetv2_e2e.yml:179-256; AUTO_FOCUS / DO_PRUNING / CHIP_HYPERPARAMS are
        # not in the yml and keep configs/faster/default_configs.py's values.  NMS -1 reaches only the soft-NMS's
        # linear / hard branches; the aggregation runs the Gaussian one (method 2), which reads NMS_SIGMA.
        test = S(SCALES=[(1400, 2000), (800, 1280), (480, 512)], BATCH_IMAGES=[2, 2, 4], MAX_PER_IMAGE=200,
                 VALID_RANGES=[(-1, 90), (32, 180), (75, -1)], AUTO_FOCUS=False, DO_PRUNING=[False, False, False],
                 CHIP_HYPERPARAMS=[(-1, -1, -1), (-1, -1, -1), (-1, -1, -1)], NMS=-1, NMS_SIGMA=0.55,
                 RPN_NMS_THRESH=0.7, RPN_PRE_NMS_TOP_N=6000, RPN_POST_NMS_TOP_N=300, RPN_MIN_SIZE=0)
    else:
        raise ValueError("default_config: network must be 'resnet101' or 'mobilenetv2', not %r" % (network,))
    num_classes, name = 81, "coco"
    if dataset == "pascal_voc":
        if network != "resnet101":
            raise ValueError("default_config: the PASCAL VOC config is a ResNet-101 one, not %r" % (network,))
        # configs/faster/sniper_res101_e2e_pascal_voc.yml: PIXEL_MEANS :17-20, the anchors :21-39, NUM_CLASSES :41;
        # TEST :177-225 (MAX_PER_IMAGE :177, SCALES :180-183, BATCH_IMAGES :186-189, VALID_RANGES :204-207, NMS / sigma
        # :224-225).  AUTO_FOCUS / DO_PRUNING / CHIP_HYPERPARAMS are not in the yml and keep
        # configs/faster/default_configs.py:164-166.
        net = S(PIXEL_MEANS=[103.939, 116.779, 123.68], ANCHOR_SCALES=[2, 4, 7, 10, 13, 16, 24], ANCHOR_RATIOS=[0.5, 1, 2],
                RPN_FEAT_STRIDE=16, NUM_ANCHORS=21)
        test = S(SCALES=[(1400, 2000), (800, 1280), (480, 512)], BATCH_IMAGES=[2, 2, 4], MAX_PER_IMAGE=200,
                 VALID_RANGES=[(-1, 90), (32, 180), (75, -1)], AUTO_FOCUS=False, DO_PRUNING=[False, False, False],
                 CHIP_HYPERPARAMS=[(-1, -1, -1), (-1, -1, -1), (-1, -1, -1)], NMS=-1, NMS_SIGMA=0.55,
                 RPN_NMS_THRESH=0.7, RPN_PRE_NMS_TOP_N=6000, RPN_POST_NMS_TOP_N=300, RPN_MIN_SIZE=0)
        num_classes, name = 21, "PascalVOC"
    elif dataset != "coco":
        raise ValueError("default_config: dataset must be 'coco' or 'pascal_voc', not %r" % (dataset,))
    return S(network=net,
             TRAIN=S(SCALES=[(1400, 2000), (800, 1280), (-1, 512)], VALID_RANGES=[(-1, 80), (32, 150), (120, -1)],
                     CPP_CHIPS=True, USE_NEG_CHIPS=neg, RPN_BATCH_SIZE=256, RPN_FG_FRACTION=0.5,
                     RPN_POSITIVE_OVERLAP=0.5, RPN_NEGATIVE_OVERLAP=0.4, BATCH_IMAGES=16, AUTO_FOCUS=autofocus,
                     AUTO_FOCUS_DC_LOW=5, AUTO_FOCUS_SMALL_THRESH=64, AUTO_FOCUS_DC_HIGH=90, FLIP=True,
                     FG_THRESH=0.5, BG_THRESH_HI=0.5, BG_THRESH_LO=0.0, BBOX_REGRESSION_THRESH=0.5,
                     BBOX_NORMALIZATION_PRECOMPUTED=True, BBOX_MEANS=[0.0, 0.0, 0.0, 0.0],
                     BBOX_STDS=[0.1, 0.1, 0.2, 0.2]),
             TEST=test,
             CLASS_AGNOSTIC=True,
             dataset=S(NUM_CLASSES=num_classes, dataset=name))
