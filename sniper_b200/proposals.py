"""RPN proposals into the training roidb: the loading half of negative-chip mining (TRAIN.USE_NEG_CHIPS).

Mirror of the reference's `imdb.load_rpn_data`, `load_rpn_roidb`, `rpn_roidb`, `create_roidb_from_box_list` and the
static `merge_roidbs` (lib/dataset/imdb.py:81-200, 399-419): same file names (`<name>_rpn.pkl` in, the
`<name>_rpn_after_nms.pkl` cache), field names and dtypes.  The proposal file is what
`tester.imdb_proposal_extraction_wrapper` writes (one float32 [n, 5] array per image); pickles written by Python 2
load too.  What changes is where the NMS runs:

  reference                                           here
  nmsp (numpy, O(N^2) per image) in a Pool(32)        `sniper_proposal_nms_batched`: one CTA per image, one launch
                                                      per chunk of images, same keep lists
  bbox_overlaps_cython                                `host.bbox_overlaps` (bit-identical to it)

The roidb that `rpn_roidb(gt_roidb, append_gt=True)` returns is what `iterator.MNIteratorE2E` with USE_NEG_CHIPS reads:
GT rows first, then the proposals with gt_classes 0, gt_overlaps / max_overlaps / max_classes from their best GT
overlap.  As in the reference, a proposal that coincides with a GT box gets max_overlaps == 1 and the iterator then
treats it as one more GT box.  One deliberate difference: the reference's merge tests `'proposal_scores' in a` on the
roidb list instead of its entries, so its merged `proposal_scores` keeps only the GT rows' 10s; here the proposal
rows' scores follow them, one score per box.
"""
import os
import pickle

import numpy as np
import torch

from . import host, ops, recall

NMS_CHUNK = 4096          # images per device launch


def _load_pickle(path):
    with open(path, 'rb') as f:
        return pickle.load(f, encoding='latin1')


def nms_keeps(box_list, device="cuda", chunk=NMS_CHUNK):
    """nmsp (IoU 0.7) of every array of box_list ([n, 5] float32 x1, y1, x2, y2, score) -> list of kept-row index
    arrays in nmsp's keep order.  The images go to the device `chunk` at a time."""
    keeps = []
    for c0 in range(0, len(box_list), chunk):
        part = box_list[c0:c0 + chunk]
        for k, b in enumerate(part):
            if b.dtype != np.float32 or b.ndim != 2 or b.shape[1] != 5:
                raise ValueError("proposals of image %d: expected float32 [n, 5] rows, got %s %s"
                                 % (c0 + k, b.dtype, b.shape))
        sizes = np.array([b.shape[0] for b in part], dtype=np.int64)
        offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
        flat = np.concatenate(part, 0) if offsets[-1] else np.zeros((0, 5), np.float32)
        dets = torch.from_numpy(np.ascontiguousarray(flat)).to(device)
        keep, counts = ops.proposal_nms_batched(dets, offsets)
        keeps += [keep[offsets[k]:offsets[k] + counts[k]].astype(np.int64) for k in range(len(part))]
    return keeps


class IMDB(object):
    """The proposal-loading methods of the reference's IMDB for a dataset `name` (e.g. 'coco_train2014', the prefix of
    its proposal files) with `num_classes` classes, background included."""

    def __init__(self, name, num_classes, device="cuda"):
        self.name, self.num_classes, self.device = name, num_classes, device

    def load_rpn_data(self, proposal_path='data/proposals', full=False):
        """(boxes, maps): the NMS-ed proposals of every image, read from the `_rpn_after_nms.pkl` cache when it exists,
        otherwise computed from `_rpn.pkl` and cached."""
        rpn_file = os.path.join(proposal_path, self.name + '_rpn.pkl')
        nms_cache_file = os.path.join(proposal_path, self.name + '_rpn_after_nms.pkl')
        if os.path.isfile(nms_cache_file):
            boxes, maps = _load_pickle(nms_cache_file)
            return boxes, maps
        if not os.path.exists(rpn_file):
            raise FileNotFoundError('rpn data not found at {}'.format(rpn_file))
        ttboxes = [np.array(b) for b in _load_pickle(rpn_file)]
        keeps = nms_keeps(ttboxes, device=self.device)
        boxes = [t[k] for t, k in zip(ttboxes, keeps)]
        maps = []
        with open(nms_cache_file, 'wb') as f:
            pickle.dump([boxes, maps], f, pickle.HIGHEST_PROTOCOL)
        return boxes, maps

    def load_rpn_roidb(self, gt_roidb, proposal_path):
        box_list, mapping_list = self.load_rpn_data(proposal_path)
        return self.create_roidb_from_box_list(box_list, mapping_list, gt_roidb)

    def rpn_roidb(self, gt_roidb, append_gt=False, cfg='', proposal_path='proposals'):
        """The proposal roidb, appended to the GT roidb (in place, as the reference does) when append_gt."""
        self.cfg = cfg
        rpn = self.load_rpn_roidb(gt_roidb, proposal_path)
        return IMDB.merge_roidbs(gt_roidb, rpn) if append_gt else rpn

    def create_roidb_from_box_list(self, box_list, mapping_list, gt_roidb):
        """One roidb entry per image from its proposals ([n, 5] rows with the score last): every proposal is labelled
        with the class of the GT box it overlaps most (overlap > 0), as gt_overlaps[n, num_classes] float32."""
        if len(box_list) != len(gt_roidb):
            raise ValueError('number of boxes matrix must match number of images')
        roidb = []
        for i, g in enumerate(gt_roidb):
            boxes = box_list[i]
            if boxes.ndim != 2 or boxes.shape[1] != 5:
                raise ValueError("proposals of image %d: expected [n, 5] rows with the score last" % i)
            scores, boxes = boxes[:, -1], boxes[:, :4]
            num_boxes = boxes.shape[0]
            overlaps = np.zeros((num_boxes, self.num_classes), dtype=np.float32)
            if g['boxes'].size > 0:
                gt_classes = g['gt_classes']
                gt_overlaps = host.bbox_overlaps(boxes.astype(np.float64), g['boxes'].astype(np.float64))
                argmaxes = gt_overlaps.argmax(axis=1)
                maxes = gt_overlaps.max(axis=1)
                I = np.where(maxes > 0)[0]
                overlaps[I, gt_classes[argmaxes[I]]] = maxes[I]
            roi_rec = {'image': g.get('image'), 'height': g['height'], 'width': g['width'],
                       'boxes': boxes,
                       'gt_classes': np.zeros((num_boxes,), dtype=np.int32),
                       'gt_overlaps': overlaps,
                       'max_classes': overlaps.argmax(axis=1),
                       'max_overlaps': overlaps.max(axis=1),
                       'flipped': False,
                       'proposal_scores': scores}
            roidb.append(roi_rec)
        return roidb

    def evaluate_recall(self, roidb, candidate_boxes=None, thresholds=None):
        """Proposal recall per GT area range of every entry of roidb, which gives the image count this class lacks
        (recall.evaluate_recall): the reference's info string, printed and returned."""
        return recall.evaluate_recall(roidb, candidate_boxes, thresholds, num_images=len(roidb),
                                      device=self.device)

    @staticmethod
    def merge_roidbs(a, b):
        """Appends b[i]'s rows to a[i]'s (in place) and returns a.  Entries without `proposal_scores` (GT) score 10."""
        if len(a) != len(b):
            raise ValueError("merge_roidbs: %d and %d entries" % (len(a), len(b)))
        for ra, rb in zip(a, b):
            for r in (ra, rb):
                if 'proposal_scores' not in r:
                    r['proposal_scores'] = 10 * np.ones(r['boxes'].shape[0])
            ra['boxes'] = np.vstack((ra['boxes'], rb['boxes']))
            ra['gt_classes'] = np.hstack((ra['gt_classes'], rb['gt_classes']))
            ra['gt_overlaps'] = np.vstack((ra['gt_overlaps'], rb['gt_overlaps']))
            ra['max_classes'] = np.hstack((ra['max_classes'], rb['max_classes']))
            ra['max_overlaps'] = np.hstack((ra['max_overlaps'], rb['max_overlaps']))
            ra['proposal_scores'] = np.hstack((ra['proposal_scores'], rb['proposal_scores']))
        return a
