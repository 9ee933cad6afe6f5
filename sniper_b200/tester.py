"""AutoFocus multi-scale inference: the test iterator, `Tester` and the scale pyramid driver.

Host-side mirror of `lib/iterators/MNIteratorTestAutoFocus.py` (:13-141), `lib/inference.py` `Tester.detect` (:100-139),
`Tester.get_detections` (:232-370), `Tester.aggregate` (:152-230, in `inference.aggregate`) and
`imdb_detection_wrapper` / `detect_scale_worker` (:400-528), TEST.CONCURRENT_JOBS included: same names, argument
meaning and returned structures (`all_boxes[class][image][chip]`, `all_maps[image][chip]`).  What changes is where the
arithmetic runs:

  reference                                             here
  cv2 crop / resize / pad in a thread pool              one `sniper_chip_input_hw` launch per batch (uint8 crops over PCIe)
  MXNet module forward (RPN, MultiProposal op on host)  `SniperResNet101.forward_inference` (device MultiProposal)
  bbox_pred / clip / rescale in numpy per chip          the same numpy code (`inference.detect_postprocess`), or with
                                                        backend="device" one `sniper_detect_post` launch per batch into
                                                        a device run buffer (no detection crosses to the host before
                                                        the soft-NMS has run)
  per-(image, class) cpu_soft_nms in a Pool(32)         `inference.aggregate`, one path for both backends: ONE
                                                        `sniper_soft_nms_batched` launch for the whole run
  FocusChips with OpenCV                                `chips_inference.add_chips`; with backend="device" the
                                                        FocusPixel maps stay on the GPU and one `sniper_focus_chips`
                                                        launch per scale finds the chips of all of them

The proposal extraction of main_test.py with TEST.EXTRACT_PROPOSALS -- `MNIteratorTest`, `Tester.get_proposals` /
`extract_proposals` and `imdb_proposal_extraction_wrapper` (lib/iterators/MNIteratorTest.py, lib/inference.py:76-98,
372-409, 532-610) -- runs `SniperResNet101.forward_rpn` on whole images; `proposals.py` loads its output into the
training roidb for negative-chip mining.

roidb entries need `width`, `height`, `image_data` (decoded BGR uint8 [H,W,3]; this image has no OpenCV to decode files)
or an `image_loader`; `inference_crops` is initialised to the full image like the reference does.
"""
import math
import os
import pickle
import time
from typing import Protocol

import numpy as np
import torch

from . import chips_inference, inference
from ._lib import check, lib


class _ImageCanvas(object):
    """Pixel stage of the test iterators: uint8 source rectangles, resized by their scale and zero-padded into an
    SH x SW canvas minus PIXEL_MEANS by one `sniper_chip_input_hw` launch per batch.  The canvas geometry follows the
    backbone's stride, config.network.RPN_FEAT_STRIDE (`_canvas_size`)."""

    def _init_canvas(self, config, device, image_loader):
        self.stride = int(config.network.RPN_FEAT_STRIDE)
        self.device = torch.device(device)
        self.image_loader = image_loader
        self.on_gpu = self.device.type == "cuda"        # host-only use (tests of the batching logic): no canvas is built
        self.means = torch.tensor(list(config.network.PIXEL_MEANS), dtype=torch.float32,
                                  device=self.device if self.on_gpu else "cpu")
        self._pix = None

    def _image(self, r):
        if 'image_data' in r:
            return r['image_data']
        if self.image_loader is None:
            raise RuntimeError("roidb entry has no 'image_data' and no image_loader was given (no OpenCV in this image)")
        return self.image_loader(r['image'])

    def _canvas(self, rects, scales, SH, SW):
        """rects: (image, y1, y2, x1, x2, flip) per batch entry.  Returns dict(data [n,3,SH,SW], im_info [n,3] =
        (resized h, resized w, scale)) on the device, or the launch's inputs (pixels, table, canvas, im_info) on a
        host-only iterator."""
        n = len(rects)
        need = sum(max(y2 - y1, 0) * max(x2 - x1, 0) * 3 for _, y1, y2, x1, x2, _ in rects)
        pix = np.empty(need, dtype=np.uint8)
        table = np.zeros((n, 8), dtype=np.int64)
        im_info = np.zeros((n, 3), dtype=np.float32)
        off = 0
        for k, ((im, y1, y2, x1, x2, flip), scale) in enumerate(zip(rects, scales)):
            h, w = max(y2 - y1, 0), max(x2 - x1, 0)
            m = h * w * 3
            if m:
                pix[off:off + m].reshape(h, w, 3)[...] = im[y1:y2, x1:x2, :3]
            dh, dw = int(np.rint(h * scale)), int(np.rint(w * scale))              # cv2.resize dsize = cvRound(...)
            dh, dw = min(dh, SH), min(dw, SW)
            table[k] = [off, h, w, dh, dw, 1 if flip else 0, int(np.float64(scale).view(np.int64)), 0]
            im_info[k] = [dh, dw, scale]
            off += m
        if not self.on_gpu:
            return dict(pixels=pix, table=table, canvas=(SH, SW), im_info=torch.from_numpy(im_info))
        dev = self.device
        if self._pix is None or self._pix.numel() < need:
            self._pix = torch.empty(int(need * 1.25) + 4096, dtype=torch.uint8, device=dev)
        self._pix[:need].copy_(torch.from_numpy(pix), non_blocking=True)
        tab = torch.from_numpy(table).to(dev)
        data = torch.empty(n, 3, SH, SW, device=dev)
        check(lib().sniper_chip_input_hw(self._pix.data_ptr(), tab.data_ptr(), self.means.data_ptr(), data.data_ptr(), n, SH,
                                         SW, torch.cuda.current_stream().cuda_stream))
        return dict(data=data, im_info=torch.from_numpy(im_info).to(dev), im_info_host=im_info)


class DetectionNetwork(Protocol):
    """What `Tester`, the test iterators and `imdb_detection_wrapper` read from a network (`model.SniperResNet101`,
    `model_mnv2.SniperMobileNetV2`):

      device             where the batches are built and the detections are kept
      feat_stride        the backbone's output stride (16 / 32); it must equal the config's network.RPN_FEAT_STRIDE,
                         from which the iterators size their canvases
      af                 the FocusPixel branch, or None for a network without one (then no FocusPixel map is asked for)
      forward_inference  (data [B,3,H,W], im_info [B,3], autofocus=False) -> (rois [B*R,5], rpn scores [B*R],
                         cls_prob [B*R,K], bbox_pred [B*R,4], + the FocusPixel map with autofocus=True); bbox_pred is
                         class-agnostic: every class takes its box from columns 0:4, as the reference's get_detections"""
    device: object
    feat_stride: int
    af: object

    def forward_inference(self, data, im_info, autofocus=False): ...


def _canvas_size(h, w, stride=16):
    """A canvas that survives a backbone of output stride `stride`: the conv kernel wants every layer's output width to
    be a multiple of 8 pixels (so the canvas width a multiple of 8 * stride: 128 at stride 16, 256 at stride 32); heights
    are free (a multiple of 32, which every stride-16 or stride-32 layer divides)."""
    hm, wm = max(32, stride), 8 * stride
    return -(-h // hm) * hm, -(-w // wm) * wm


class MNIteratorTestAutoFocus(_ImageCanvas):
    """MNIteratorTestAutoFocus(roidb, config, test_scale, batch_size, ...): batches of chips of one test scale, sorted by
    area and grouped by orientation (reset :88-141); a batch is padded to its largest resized chip (_get_batch :36-78)."""

    def __init__(self, roidb, config, test_scale, batch_size=4, threads=8, nGPUs=1, pad_rois_to=400, crop_size=(512, 512),
                 num_classes=None, device="cuda:0", image_loader=None):
        self.roidb, self.cfg, self.test_scale = roidb, config, test_scale
        self.batch_size = batch_size
        self.data_name = ['data', 'im_info', 'im_ids', 'chip_ids']
        self._init_canvas(config, device, image_loader)
        self.reset()

    def set_scale(self, scale):
        self.test_scale = scale

    def reset(self):
        self.cur_i = 0
        self.crop2im = {}
        widths, heights = [], []
        crop_counter = 0
        for i, r in enumerate(self.roidb):
            local_crop_mapping = {}
            for local_counter, crop in enumerate(r['inference_crops']):
                widths.append(crop[2] - crop[0])
                heights.append(crop[3] - crop[1])
                self.crop2im[crop_counter] = i
                local_crop_mapping[crop_counter] = local_counter
                crop_counter += 1
            r['crop_mapping'] = local_crop_mapping
        self.n_chips = crop_counter
        if crop_counter == 0:
            self.inds, self.size = np.zeros(0, dtype=int), 0
            return
        widths, heights = np.array(widths, dtype=np.float64), np.array(heights, dtype=np.float64)
        order = (widths * heights).argsort()                   # sort based on area
        widths, heights = widths[order], heights[order]
        horz_inds = np.where(widths >= heights)[0]
        vert_inds = np.where(widths < heights)[0]
        bs = self.batch_size
        if horz_inds.shape[0] % bs > 0:
            extra = bs - (horz_inds.shape[0] % bs)
            horz_inds = np.hstack((horz_inds, horz_inds[-extra:]))
        if vert_inds.shape[0] % bs > 0:
            extra = bs - (vert_inds.shape[0] % bs)
            vert_inds = np.hstack((vert_inds, vert_inds[-extra:]))
        inds = np.hstack((horz_inds, vert_inds)).astype(int)
        if inds.shape[0] % bs > 0:                             # a group smaller than its padding request
            extra = bs - (inds.shape[0] % bs)
            inds = np.hstack((inds, np.resize(inds[-extra:], extra)))
        self.inds = order[inds]
        self.size = len(self.inds)

    def __iter__(self):
        return self

    def get_batch_size(self):
        return self.batch_size

    def __next__(self):
        if self.cur_i >= self.size:
            raise StopIteration
        chip_ids = [int(self.inds[i % self.size]) for i in range(self.cur_i, self.cur_i + self.batch_size)]
        im_ids = [self.crop2im[c] for c in chip_ids]
        self.cur_i += self.batch_size
        return self._get_batch([self.roidb[i] for i in im_ids], chip_ids, im_ids)

    next = __next__

    def _get_batch(self, roidb, chip_ids, im_ids):
        n = len(roidb)
        max_size = [0, 0]
        rects, scales, local_chip_ids = [], [], np.zeros(n)
        for i, r in enumerate(roidb):
            scale = chips_inference.image_scale(r['width'], r['height'], self.test_scale)
            cchip_id = r['crop_mapping'][chip_ids[i]]
            cur_chip = r['inference_crops'][cchip_id]
            local_chip_ids[i] = cchip_id
            max_size[0] = max(max_size[0], int(math.ceil((cur_chip[3] - cur_chip[1]) * scale)))
            max_size[1] = max(max_size[1], int(math.ceil((cur_chip[2] - cur_chip[0]) * scale)))
            im = self._image(r)
            y1, y2 = max(int(cur_chip[1]), 0), min(int(cur_chip[3]), im.shape[0])     # worker_autofocus :60-62
            x1, x2 = max(int(cur_chip[0]), 0), min(int(cur_chip[2]), im.shape[1])
            rects.append((im, y1, y2, x1, x2, False))
            scales.append(scale)
        out = self._canvas(rects, scales, *_canvas_size(max_size[0], max_size[1], self.stride))
        out.update(im_ids=np.array(im_ids, dtype=int), chip_ids=local_chip_ids.astype(int), scales=np.array(scales))
        return out


class MNIteratorTest(_ImageCanvas):
    """MNIteratorTest(roidb, config, test_scale, batch_size, ...) (lib/iterators/MNIteratorTest.py): batches of whole
    images at one test scale, horizontal images first, then vertical ones (reset :50-66).  Each image is resized by
    `chips_inference.image_scale`.  The canvas is the test scale (swapped for vertical images) rounded up to the conv
    kernel's multiples, the same for every batch of an orientation, so an image's proposals do not depend on which
    images share its batch.  (The score-0 filler rows MultiProposal appends when an image has fewer than 300 proposals
    do: their boxes follow the image's position in the batch, as the reference's rand() boxes follow the call order.)"""

    def __init__(self, roidb, config, test_scale, batch_size=4, threads=8, nGPUs=1, pad_rois_to=400, crop_size=None,
                 num_classes=None, device="cuda:0", image_loader=None):
        self.roidb, self.cfg, self.test_scale = roidb, config, test_scale
        self.batch_size = batch_size
        self.data_name = ['data', 'im_info', 'im_ids']
        self._init_canvas(config, device, image_loader)
        self.reset()

    def set_scale(self, scale):
        self.test_scale = scale

    def reset(self):
        """self.inds: image indices in batch order; a group that does not fill its last batch repeats its first image."""
        self.cur_i = 0
        widths = np.array([r['width'] for r in self.roidb])
        heights = np.array([r['height'] for r in self.roidb])
        bs = self.batch_size
        groups = []
        for g in (np.where(widths >= heights)[0], np.where(widths < heights)[0]):
            if g.shape[0] % bs > 0:
                g = np.hstack((g, g[np.zeros(bs - g.shape[0] % bs, dtype=int)]))
            groups.append(g)
        self.inds = np.hstack(groups).astype(int)
        self.size = len(self.inds)

    def __iter__(self):
        return self

    def get_batch_size(self):
        return self.batch_size

    def __next__(self):
        if self.cur_i >= self.size:
            raise StopIteration
        im_ids = [int(self.inds[i % self.size]) for i in range(self.cur_i, self.cur_i + self.batch_size)]
        self.cur_i += self.batch_size
        return self._get_batch([self.roidb[i] for i in im_ids], im_ids)

    next = __next__

    def _get_batch(self, roidb, im_ids):
        hor = roidb[0]['width'] >= roidb[0]['height']
        max_size = (self.test_scale[0], self.test_scale[1]) if hor else (self.test_scale[1], self.test_scale[0])
        rects, scales = [], []
        for r in roidb:
            im = self._image(r)
            rects.append((im, 0, im.shape[0], 0, im.shape[1], bool(r.get('flipped', False))))
            scales.append(chips_inference.image_scale(r['width'], r['height'], self.test_scale))
        out = self._canvas(rects, scales, *_canvas_size(max_size[0], max_size[1], self.stride))
        out.update(im_ids=np.array(im_ids, dtype=int), scales=np.array(scales))
        return out


class Tester(object):
    """Tester(module, imdb, roidb, test_iter, cfg, ...): `module` = a `DetectionNetwork` (`SniperResNet101`,
    `SniperMobileNetV2`) for the detections, or a network with `forward_rpn` for the proposals."""

    def __init__(self, module, imdb, roidb, test_iter, cfg, rcnn_output_names=None, rpn_output_names=None, logger=None,
                 batch_size=None, num_classes=None):
        self.net, self.imdb, self.roidb, self.test_iter, self.cfg = module, imdb, roidb, test_iter, cfg
        self.batch_size = batch_size
        self.num_images = len(roidb)
        self.num_classes = num_classes or (imdb.num_classes if imdb is not None else cfg.dataset.NUM_CLASSES)
        self.detect_time = self.post_time = 0.0

    def get_proposals(self, batch, scales):
        """(scores, rois, batch, im_ids) of one batch (:76-98) from `net.forward_rpn`: per image its rpn scores [R] and
        boxes [R,4] in ORIGINAL-image scale (rois / float32 im_info scale)."""
        rois, rscores = self.net.forward_rpn(batch['data'], batch['im_info'])
        rois, rscores = rois.cpu().numpy(), rscores.cpu().numpy().reshape(-1)
        scores, boxes = [], []
        for idx in range(batch['data'].shape[0]):
            cids = np.where(rois[:, 0] == idx)[0]
            boxes.append(rois[cids, 1:] / np.float32(scales[idx]))
            scores.append(rscores[cids])
        return scores, boxes, batch, batch['im_ids']

    def extract_proposals(self, n_proposals=300, cache_name='cache', vis=False, vis_ext='.png'):
        """all_boxes[image] = float32 [n_proposals, 5] (x1, y1, x2, y2, score) (:372-409): every image's first
        n_proposals rows, in original-image coordinates."""
        all_boxes = [[] for _ in range(self.num_images)]
        for batch in self.test_iter:
            scales = batch['im_info'].cpu().numpy()[:, 2]
            t0 = time.time()
            scores, boxes, _, im_ids = self.get_proposals(batch, scales)
            self.detect_time += time.time() - t0
            t0 = time.time()
            for cscores, cboxes, im_id in zip(scores, boxes, im_ids):
                all_boxes[im_id] = np.hstack((cboxes[0:n_proposals, 0:4],
                                              cscores[0:n_proposals, np.newaxis])).astype(np.float32)
            self.post_time += time.time() - t0
        return all_boxes

    def detect(self, batch, scales=None):
        """(scores, boxes, data, im_ids, maps, chip_ids) of one batch (:100-139): scores [R,K] and boxes [R,4] per chip,
        boxes in ORIGINAL-image scale relative to the chip origin."""
        want_map = bool(getattr(self.cfg.TEST, "AUTO_FOCUS", False)) and self.net.af is not None
        out = self.net.forward_inference(batch['data'], batch['im_info'], autofocus=want_map)
        rois, _, cls_prob, deltas = out[:4]
        B = batch['data'].shape[0]
        scores, preds = inference.detect_postprocess(rois.cpu().numpy(), cls_prob.cpu().numpy(), deltas.cpu().numpy(),
                                                     batch['im_info'].cpu().numpy(), B)
        maps = self._chip_maps(out[4].cpu().numpy(), batch['im_info'].cpu().numpy()) if want_map else []
        return scores, preds, batch, batch['im_ids'], maps, batch['chip_ids']

    def _chip_maps(self, fm, im_info):
        """The FocusPixel map of each chip of a batch: fm [B,H,W] covers the canvas, which is padded to the batch
        maximum, so chip idx's own map is its first ceil(resized height / stride) x ceil(resized width / stride) cells."""
        s = float(self.net.feat_stride)
        return [fm[idx, :int(math.ceil(im_info[idx, 0] / s)), :int(math.ceil(im_info[idx, 1] / s))].copy()
                for idx in range(fm.shape[0])]

    def get_detections(self, cls_thresh=1e-3, cache_name='cache', evaluate=False, vis=False, vis_path=None,
                       do_pruning=False, autofocus=False, vis_ext='.png', backend="host", scale_index=0):
        """(all_boxes, all_maps) (:232-370): all_boxes[j][im][chip] = [n,5], all_maps[im][chip] = (None, FocusPixel map).
        backend="device": all_boxes is the scale's `inference.DeviceDetections` instead (rows already through
        TEST.VALID_RANGES[scale_index]); see `_get_detections_device`."""
        if backend == "device":
            return self._get_detections_device(cls_thresh, do_pruning, autofocus, scale_index)
        if backend != "host":
            raise ValueError("get_detections: backend must be 'host' or 'device', not %r" % (backend,))
        n_chips = [len(r['inference_crops']) for r in self.roidb]
        all_boxes = [[[np.zeros((0, 5), np.float32) for _ in range(n_chips[i])] for i in range(self.num_images)]
                     for _ in range(self.num_classes)]
        all_maps = [[[] for _ in range(n_chips[i])] for i in range(self.num_images)]
        for batch in self.test_iter:
            t0 = time.time()
            scores, boxes, _, im_ids, maps, chip_ids = self.detect(batch)
            if torch.device(self.net.device).type == "cuda":
                torch.cuda.synchronize()
            self.detect_time += time.time() - t0
            t0 = time.time()
            for i, (cscores, cboxes, im_id, chip_id) in enumerate(zip(scores, boxes, im_ids, chip_ids)):
                if autofocus and maps:
                    all_maps[im_id][chip_id] = (None, maps[i])
                # score threshold per class; with do_pruning also: project back to the image and drop detections cut
                # by a chip border (:335-351), for all classes in one pass
                r = self.roidb[im_id]
                prune = (r['inference_crops'][chip_id], r['width'], r['height']) if do_pruning else None
                dets = inference.threshold_detections(cscores, cboxes, self.num_classes, cls_thresh, prune=prune)
                for j in range(1, self.num_classes):
                    all_boxes[j][im_id][chip_id] = dets[j]
            self.post_time += time.time() - t0
        return all_boxes, all_maps

    def _get_detections_device(self, cls_thresh, do_pruning, autofocus, scale_index):
        """The batches of the scale with the detections kept on the device: `forward_inference`, then `ops.detect_post`
        on its output tensors, fed by the batch's chip table.  all_maps is a `chips_inference.DeviceFocusMaps`: each
        batch's FocusPixel map tensor stays on the device (no map is copied to the host) for `add_chips` to run
        `ops.focus_chips` on; maps[i][j] still gives a host copy."""
        want_map = bool(getattr(self.cfg.TEST, "AUTO_FOCUS", False)) and self.net.af is not None
        dets = inference.DeviceDetections(self.net.device)
        all_maps = chips_inference.DeviceFocusMaps([len(r['inference_crops']) for r in self.roidb], self.net.feat_stride)
        seen = set()
        t0 = time.time()
        for batch in self.test_iter:
            out = self.net.forward_inference(batch['data'], batch['im_info'], autofocus=want_map)
            rois, _, cls_prob, deltas = out[:4]
            table = inference.chip_table(self.roidb, batch['im_ids'], batch['chip_ids'], do_pruning,
                                         self.cfg.TEST.VALID_RANGES[scale_index], seen)
            dets.append(rois, cls_prob, deltas, batch['im_info'], table, cls_thresh=cls_thresh, scale=scale_index)
            if want_map and autofocus:
                all_maps.add(out[4], batch['im_info_host'], batch['im_ids'], batch['chip_ids'])
        dets.finish()
        self.detect_time += time.time() - t0
        return dets, all_maps

    def aggregate(self, scale_cls_dets, vis=False, cache_name='cache', vis_path=None, vis_name=None, pre_nms_db_divide=10,
                  vis_ext='.png', backend="device"):
        t = self.cfg.TEST
        return inference.aggregate(scale_cls_dets, t.VALID_RANGES, self.num_images, self.num_classes,
                                   sigma=getattr(t, "NMS_SIGMA", 0.55), nms_thresh=getattr(t, "NMS", 0.3),
                                   max_per_image=t.MAX_PER_IMAGE, backend=backend,
                                   device=str(self.net.device) if self.net is not None else "cuda")


def job_blocks(num_images, jobs):
    """The image range [lo, hi) of each of `jobs` concurrent test jobs, in job order, as the reference's wrappers split
    the roidb for TEST.CONCURRENT_JOBS > 1 (:457-461, 568-572): im_per_job = ceil(N / jobs) images per job, so the
    trailing blocks can be short or empty (N = 5, jobs = 4: 2, 2, 1 and 0 images)."""
    if int(jobs) != jobs or jobs < 1:
        raise ValueError("concurrent_jobs must be a positive integer, not %r" % (jobs,))
    per = -(-num_images // jobs)
    return [(min(per * j, num_images), min(per * (j + 1), num_images)) for j in range(jobs)]


def _world(group):
    if group is None:
        return 1, 0
    return torch.distributed.get_world_size(group), torch.distributed.get_rank(group)


def _same_on_all_ranks(value, what, group):
    """Collective: raises ValueError on every rank of `group` unless `value` is equal on all of them."""
    got = [None] * _world(group)[0]
    torch.distributed.all_gather_object(got, value, group=group)
    if any(v != got[0] for v in got):
        raise ValueError("the ranks' %s differ: %s" % (what, ", ".join("rank %d: %r" % (r, v) for r, v in enumerate(got))))


def _test_roidb_digest(roidb):
    """iterator.roidb_digest of a test roidb, whose entries may carry no GT boxes."""
    from .iterator import roidb_digest
    return roidb_digest([r if 'boxes' in r else dict(r, boxes=np.zeros((0, 4))) for r in roidb])


def _concurrent_jobs(roidb, jobs, group, run_job):
    """Runs run_job(block) -> (result, stats) on the roidb block of every job (`job_blocks`) and yields (result, job
    stats) in job order.  A job's stats are dict(images=(lo, hi), rank=<rank it ran on>) plus run_job's own; an empty
    block runs nothing and yields (None, dict(images, rank, scales=[])).

    With a process group of W ranks, job j runs on rank j mod W, W jobs at a time.  Each job's result then goes to
    rank 0 on its own (point to point, in job order), so rank 0 holds at most one received result beyond what its
    caller has merged, and nothing is all-gathered.  Rank 0 yields every job; another rank yields (None, stats) for its
    own jobs only.  Before any work the ranks compare the roidb's digest and `jobs`; before each round's results move
    they share every job's success or failure, so an exception on one rank (a detect_post capacity error, say) raises
    RuntimeError with that rank's message on every rank instead of leaving the others waiting in a collective."""
    world, rank = _world(group)
    if world > 1:
        _same_on_all_ranks((_test_roidb_digest(roidb), int(jobs)), "test roidbs and concurrent_jobs", group)
    blocks = job_blocks(len(roidb), jobs)
    dist = torch.distributed
    for first in range(0, jobs, world):
        j = first + rank
        result = st = err = failure = None
        if j < jobs:
            lo, hi = blocks[j]
            st = dict(images=(lo, hi), rank=rank, scales=[])
            if hi > lo:
                try:
                    result, job_st = run_job(roidb[lo:hi])
                    st.update(job_st)
                except Exception as e:
                    if world == 1:
                        raise
                    err, failure = "%s: %s" % (type(e).__name__, e), e
        if world > 1:
            errs = [None] * world
            dist.all_gather_object(errs, err, group=group)
            bad = [(r, e) for r, e in enumerate(errs) if e is not None]
            if bad:
                raise RuntimeError("; ".join("concurrent test job %d (images %d:%d) failed on rank %d: %s"
                                             % ((first + r,) + tuple(blocks[first + r]) + (r, e)) for r, e in bad)
                                   ) from failure
        for k in range(first, min(first + world, jobs)):
            owner = k - first
            if owner == rank:
                if rank != 0:
                    dist.send_object_list([result, st], group=group, group_dst=0)
                    result = None
                yield result, st
            elif rank == 0:
                got = [None, None]
                dist.recv_object_list(got, group=group, group_src=owner)
                yield got[0], got[1]


def _detection_job(net, config, roidb, num_classes, batch_images, device, nms_backend, detect_backend, image_loader):
    """One test job: every scale of TEST.SCALES over `roidb` in turn (FocusChips of scale i feed scale i + 1 when
    DO_PRUNING[i + 1]), then the cross-scale aggregation.  Returns (all_boxes[class][image], stats)."""
    T = config.TEST
    detections, stats = [], dict(scales=[])
    nb = batch_images or list(T.BATCH_IMAGES)
    for scale_i, (nbatch, scale) in enumerate(zip(nb, T.SCALES)):
        it = MNIteratorTestAutoFocus(roidb, config, scale, batch_size=nbatch, device=device, image_loader=image_loader)
        tester = Tester(net, None, roidb, it, config, batch_size=nbatch, num_classes=num_classes)
        t0 = time.time()
        dets, maps = tester.get_detections(do_pruning=bool(T.DO_PRUNING[scale_i]), autofocus=bool(T.AUTO_FOCUS),
                                           backend=detect_backend, scale_index=scale_i)
        st = dict(scale=tuple(scale), chips=int(it.n_chips), batches=int(it.size // max(nbatch, 1)),
                  detect_s=tester.detect_time, post_s=tester.post_time, total_s=time.time() - t0)
        if detect_backend == "device":
            st['detections_pre_nms'] = len(dets)
        if scale_i + 1 < len(T.SCALES) and T.DO_PRUNING[scale_i + 1] and T.AUTO_FOCUS:
            t1 = time.time()
            area = chips_inference.add_chips(roidb, maps, scale_i, config)
            st.update(chip_gen_s=time.time() - t1, pixels_next_scale_pct=100.0 * area[0] / max(area[1], 1e-12))
        # the per-chip lists of a scale become one list per image for the aggregation
        detections.append(dets)
        stats['scales'].append(st)
    tester = Tester(net, None, roidb, None, config, num_classes=num_classes)
    t0 = time.time()
    all_boxes = tester.aggregate(detections, backend=nms_backend)
    torch.cuda.synchronize()
    stats['nms_s'] = time.time() - t0
    return all_boxes, stats


def imdb_detection_wrapper(net, config, roidb, num_classes=None, batch_images=None, device="cuda:0", nms_backend="device",
                           imdb=None, detect_backend="host", image_loader=None, concurrent_jobs=1, group=None):
    """imdb_detection_wrapper (:436-528): every scale of TEST.SCALES in turn (FocusChips of scale i feed scale i + 1 when
    DO_PRUNING[i + 1]), then the cross-scale aggregation.
    Returns (all_boxes[class][image], stats) with per-scale chip counts / detect / post-processing seconds, the NMS
    latency and the pixel fraction processed.  detect_backend="device" keeps the detections on the GPU from the network
    to the soft-NMS (`Tester.get_detections(backend="device")`); stats then carry `detections_pre_nms` per scale.
    With an imdb (e.g. `coco.coco`, whose gt_roidb is `roidb`), the
    dataset evaluation of :526-527 follows: imdb.evaluate_detections(all_boxes), whose result goes to stats['eval']
    and its seconds to stats['eval_s'].  `net` is a `DetectionNetwork`; config is the network's own (e.g.
    iterator.default_config(network="mobilenetv2") for a SniperMobileNetV2): its RPN_FEAT_STRIDE must be the net's.
    image_loader(path) decodes the entries without 'image_data' (e.g. host.imread).

    concurrent_jobs=J > 1 is TEST.CONCURRENT_JOBS: the images are split into J blocks (`job_blocks`) and each block runs
    the whole pipeline above on its own -- its own test iterators (so chips are sorted, grouped and padded per block),
    its own add_chips and its own aggregation -- and all_boxes[j] is the jobs' lists concatenated per class in job
    order.  That is the reference's result, where the jobs' per-scale outputs are merged and then aggregated once:
    the soft-NMS solves one (image, class) problem at a time, the MAX_PER_IMAGE cut is per image and add_chips works
    per image, so no image's result depends on which block it is in.  (With the device backend a job's run keys carry
    block-local image indices; each job aggregates its own rows, no run buffer spans two jobs.)
    group=<process group of W ranks> runs job j on rank j mod W (`_concurrent_jobs`), each rank on its own `net` /
    `device`, reading only its jobs' images.  Rank 0 merges and evaluates; the other ranks return (None, stats).  The
    group is never taken from torch.distributed implicitly: a caller that evaluates on one rank of a larger group passes
    none.  With J > 1 or a group, stats holds `jobs` (per job: images (lo, hi), rank, and the per-scale `scales` and
    `nms_s` of that job) instead of `scales` / `nms_s`; `eval` / `eval_s` stay as above, on rank 0."""
    if int(config.network.RPN_FEAT_STRIDE) != int(net.feat_stride):
        raise ValueError("imdb_detection_wrapper: config.network.RPN_FEAT_STRIDE is %s, the network's stride is %s"
                         % (config.network.RPN_FEAT_STRIDE, net.feat_stride))
    job_blocks(len(roidb), concurrent_jobs)
    for r in roidb:
        r['inference_crops'] = np.array([[0, 0, r['width'], r['height']]])

    def run_job(block):
        return _detection_job(net, config, block, num_classes, batch_images, device, nms_backend, detect_backend,
                              image_loader)
    if concurrent_jobs == 1 and group is None:
        all_boxes, stats = run_job(roidb)
    else:
        all_boxes = [[] for _ in range(num_classes or config.dataset.NUM_CLASSES)]
        stats = dict(jobs=[])
        for boxes, st in _concurrent_jobs(roidb, concurrent_jobs, group, run_job):
            stats['jobs'].append(st)
            if boxes is not None:
                for c, per_image in zip(all_boxes, boxes):
                    c += per_image
        if _world(group)[1] != 0:
            return None, stats
    if imdb is not None:
        t0 = time.time()
        stats['eval'] = imdb.evaluate_detections(all_boxes)
        stats['eval_s'] = time.time() - t0
    return all_boxes, stats


def proposal_file_name(config):
    """`<DATASET>_<test_image_set>_rpn.pkl`, the name main_test.py gives the extracted proposals (lib/inference.py:606)."""
    return '{}_{}_rpn.pkl'.format(config.dataset.dataset.upper(), config.dataset.test_image_set)


def _proposal_job(net, config, roidb, batch_images, n_proposals, device, image_loader):
    """One extraction job: RPN proposals of every image of `roidb` at every scale of TEST.SCALES, each image's rows
    stacked in scale order.  Returns (proposals[image], stats)."""
    T = config.TEST
    proposals, stats = [], dict(scales=[])
    nb = batch_images or list(T.BATCH_IMAGES)
    for nbatch, scale in zip(nb, T.SCALES):
        it = MNIteratorTest(roidb, config, scale, batch_size=nbatch, device=device, image_loader=image_loader)
        tester = Tester(net, None, roidb, it, config, batch_size=nbatch, num_classes=1)
        t0 = time.time()
        proposals.append(tester.extract_proposals(n_proposals=n_proposals))
        stats['scales'].append(dict(scale=tuple(scale), images=len(roidb), batches=int(it.size // max(nbatch, 1)),
                                    detect_s=tester.detect_time, post_s=tester.post_time, total_s=time.time() - t0))
    return [np.vstack([p[i] for p in proposals]) for i in range(len(roidb))], stats


def imdb_proposal_extraction_wrapper(net, config, roidb, save_path, batch_images=None, n_proposals=300, device="cuda:0",
                                     image_loader=None, imdb=None, concurrent_jobs=1, group=None):
    """imdb_proposal_extraction_wrapper (:559-610): RPN proposals of every image at every scale of TEST.SCALES
    (`net.forward_rpn`), each image's rows stacked in scale order, pickled as a list of float32 [n, 5] arrays to
    save_path/proposal_file_name(config) (protocol 2, readable by the reference's Python 2).  Returns
    (proposals, stats) with per-scale image / batch counts and forward / post-processing seconds.  image_loader(path)
    decodes the entries without 'image_data' (e.g. host.imread).  With an imdb (`coco.coco`, `pascal_voc.PascalVOC`
    or `proposals.IMDB`), the recall of the extracted proposals follows: imdb.evaluate_recall(roidb, candidate_boxes=
    [p[:, :4] for p in proposals]) against the GT fields of `roidb` (boxes / gt_classes / gt_overlaps), whose string
    goes to stats['recall'] and its seconds to stats['recall_s'].

    concurrent_jobs / group split the images into jobs and run them on the ranks as `imdb_detection_wrapper` does; the
    jobs' lists are concatenated in job order, which is the reference's result: it stacks each image's rows per image.
    Rank 0 writes the pickle and scores the recall; the other ranks write nothing and return (None, stats).  With
    J > 1 or a group, stats holds `jobs` (per job: images (lo, hi), rank and its `scales`) instead of `scales`."""
    job_blocks(len(roidb), concurrent_jobs)

    def run_job(block):
        return _proposal_job(net, config, block, batch_images, n_proposals, device, image_loader)
    if concurrent_jobs == 1 and group is None:
        final, stats = run_job(roidb)
    else:
        final, stats = [], dict(jobs=[])
        for props, st in _concurrent_jobs(roidb, concurrent_jobs, group, run_job):
            stats['jobs'].append(st)
            if props is not None:
                # an array received from another rank carries an unpickled float32 dtype object, equal to but not the
                # one of local arrays, which pickle would write once more: the file must not depend on the ranks
                final += [np.asarray(p, np.float32) for p in props]
        if _world(group)[1] != 0:
            return None, stats
    os.makedirs(save_path, exist_ok=True)
    with open(os.path.join(save_path, proposal_file_name(config)), 'wb') as f:
        pickle.dump(final, f, protocol=2)
    if imdb is not None:
        t0 = time.time()
        stats['recall'] = imdb.evaluate_recall(roidb, candidate_boxes=[p[:, :4] for p in final])
        stats['recall_s'] = time.time() - t0
    return final, stats
