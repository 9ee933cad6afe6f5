"""The `coco` imdb of the reference (lib/dataset/coco.py): class tables, gt_roidb and evaluate_detections.

evaluate_detections(all_boxes) writes `results/detections_<image_set>_results.json` and, unless the image set is a
test split, scores it with `sniper_b200.cocoeval` (matching and accumulation on the device), prints the per-class AP
table and returns COCOeval.stats.  all_boxes[class][i] is the [n, 5] (x1, y1, x2, y2, score) array of class `class` in
image i of `image_set_index`, which is also gt_roidb's order.

The writer is vectorised (no process pool) and keeps the reference's numbers: w = x2 - x1 + 1, boxes rounded to 1
decimal and scores to 8 with Python 2.7's round -- the exact binary value, ties away from zero -- because the reference
ran under Python 2.7 and Python 3's round differs on exact ties (x1 = 123.25 gives 123.3 under 2.7, 123.2 under 3; a
score of exactly 1/512 gives 0.00195313 under 2.7).  The file parses to the reference's list of dicts; it is not
byte-identical (Python 2's json indent added trailing spaces).

One difference in order: image_set_index is the annotation file's image order (Python 3 dicts keep insertion order),
where the reference's Python 2 dict iterated integer keys in hash order.  Scores do not depend on it.
"""
import os
import pickle
import time
from decimal import ROUND_HALF_UP, Decimal

import numpy as np
import torch

from . import recall
from .cocoeval import COCO, COCOeval


def round_py2(x, ndigits):
    """Python 2.7's round(x, ndigits) of every element of a float64 array.  Away from ties, the nearest multiple of
    10^-ndigits is rint(x * 10^ndigits) (the product's rounding error is far below the distance to the half-way point)
    and r / 10^ndigits is the double nearest to it, as 2.7's strtod of the rounded decimal gives.  Values within a
    hair of a half-way point -- the exact ties among them -- are rounded on their exact decimal expansion."""
    x = np.asarray(x, dtype=np.float64)
    s = 10.0 ** ndigits
    y = x * s
    out = np.rint(y) / s
    near = np.abs(y - np.floor(y) - 0.5) <= np.abs(y) * 1e-12 + 1e-9
    q = Decimal(1).scaleb(-ndigits)
    for i in zip(*np.nonzero(near)):
        out[i] = float(Decimal(float(x[i])).quantize(q, rounding=ROUND_HALF_UP))
    return out


class coco(object):
    def __init__(self, image_set, root_path, data_path, result_path=None, device="cuda"):
        """image_set: e.g. val2017; root_path: where cache/ goes; data_path: holds annotations/ and images/."""
        self.name = 'COCO_' + image_set
        self.image_set, self.root_path, self.data_path = image_set, root_path, data_path
        self._result_path = result_path
        self.device = device
        self.coco = COCO(self._get_ann_file())
        cats = [cat['name'] for cat in self.coco.loadCats(self.coco.getCatIds())]
        self.classes = ['__background__'] + cats
        self.num_classes = len(self.classes)
        self._class_to_ind = dict(zip(self.classes, range(self.num_classes)))
        self._class_to_coco_ind = dict(zip(cats, self.coco.getCatIds()))
        self._coco_ind_to_class_ind = dict([(self._class_to_coco_ind[cls], self._class_to_ind[cls])
                                            for cls in self.classes[1:]])
        self.image_set_index = self.coco.getImgIds()
        self.num_images = len(self.image_set_index)
        view_map = {'minival2014': 'val2014', 'sminival2014': 'val2014', 'valminusminival2014': 'val2014',
                    'test-dev2015': 'test2015'}
        self.data_name = view_map.get(image_set, image_set)
        self.eval_times = {}

    def _get_ann_file(self):
        prefix = 'instances' if 'test' not in self.image_set else 'image_info'
        return os.path.join(self.data_path, 'annotations', prefix + '_' + self.image_set + '.json')

    @property
    def cache_path(self):
        path = os.path.join(self.root_path, 'cache')
        os.makedirs(path, exist_ok=True)
        return path

    @property
    def result_path(self):
        if self._result_path and os.path.exists(self._result_path):
            return self._result_path
        return self.cache_path

    def image_path_from_index(self, index):
        filename = 'COCO_%s_%012d.jpg' % (self.data_name, index)
        image_path = os.path.join(self.data_path, 'images', self.data_name, filename)
        assert os.path.exists(image_path), 'Path does not exist: {}'.format(image_path)
        return image_path

    def gt_roidb(self):
        """One roidb entry per image (lib/dataset/coco.py:118-151), cached as <name>_gt_roidb.pkl with the image
        index lists beside it."""
        cache_file = os.path.join(self.cache_path, self.name + '_gt_roidb.pkl')
        index_file = os.path.join(self.cache_path, self.name + '_index_roidb.pkl')
        sindex_file = os.path.join(self.cache_path, self.name + '_sindex_roidb.pkl')
        if os.path.exists(cache_file) and os.path.exists(index_file):
            with open(cache_file, 'rb') as f:
                roidb = pickle.load(f, encoding='latin1')
            with open(index_file, 'rb') as f:
                self.image_set_index = pickle.load(f, encoding='latin1')
            print('{} gt roidb loaded from {}'.format(self.name, cache_file))
            return roidb
        gt_roidb = [self._load_coco_annotation(index) for index in self.image_set_index]
        valid_id = list(self.image_set_index)
        with open(cache_file, 'wb') as f:
            pickle.dump(gt_roidb, f, pickle.HIGHEST_PROTOCOL)
        with open(index_file, 'wb') as f:
            pickle.dump(valid_id, f, pickle.HIGHEST_PROTOCOL)
        with open(sindex_file, 'wb') as f:
            pickle.dump(list(range(len(valid_id))), f, pickle.HIGHEST_PROTOCOL)
        print('wrote gt roidb to {}'.format(cache_file))
        return gt_roidb

    def _load_coco_annotation(self, index):
        """lib/dataset/coco.py:153-260: the non-crowd boxes clipped to the image (x2 = x1 + max(0, w - 1)), kept when
        area > 0 and x2 >= x1, y2 >= y1, as uint16; crowd annotations only size `boxesc` (left zero)."""
        im_ann = self.coco.loadImgs(index)[0]
        width, height = im_ann['width'], im_ann['height']
        objs = self.coco.loadAnns(self.coco.getAnnIds(imgIds=index, iscrowd=False))
        objsc = self.coco.loadAnns(self.coco.getAnnIds(imgIds=index, iscrowd=True))
        b = np.array([o['bbox'] for o in objs], dtype=np.float64).reshape(-1, 4)
        area = np.array([o['area'] for o in objs], dtype=np.float64)
        x1 = np.maximum(0, b[:, 0])
        y1 = np.maximum(0, b[:, 1])
        x2 = np.minimum(width - 1, x1 + np.maximum(0, b[:, 2] - 1))
        y2 = np.minimum(height - 1, y1 + np.maximum(0, b[:, 3] - 1))
        ok = (area > 0) & (x2 >= x1) & (y2 >= y1)
        objs = [o for o, k in zip(objs, ok) if k]
        boxes = np.stack([x1, y1, x2, y2], 1)[ok].astype(np.uint16)
        gt_classes = np.array([self._coco_ind_to_class_ind[o['category_id']] for o in objs], dtype=np.int32)
        overlaps = np.zeros((len(objs), self.num_classes), dtype=np.float32)
        crowd = np.array([bool(o['iscrowd']) for o in objs], dtype=bool)
        overlaps[np.flatnonzero(~crowd), gt_classes[~crowd]] = 1.0
        overlaps[crowd, :] = -1.0
        return {'image': self.image_path_from_index(index),
                'height': height,
                'width': width,
                'boxes': boxes,
                'boxesc': np.zeros((len(objsc), 4), dtype=np.uint16),
                'gt_classes': gt_classes,
                'gt_overlaps': overlaps,
                'max_classes': overlaps.argmax(axis=1),
                'max_overlaps': overlaps.max(axis=1),
                'flipped': False}

    def evaluate_recall(self, roidb, candidate_boxes=None, thresholds=None):
        """Proposal recall per GT area range of the first num_images entries of roidb (recall.evaluate_recall): the
        reference's info string, printed and returned."""
        return recall.evaluate_recall(roidb, candidate_boxes, thresholds, num_images=self.num_images,
                                      device=self.device)

    def evaluate_detections(self, detections):
        """Writes the results json and, for a non-test image set, evaluates it; returns COCOeval.stats (None for a test
        split).  eval_times gets the seconds spent writing the json and in the evaluation."""
        res_folder = os.path.join(self.result_path, 'results')
        os.makedirs(res_folder, exist_ok=True)
        res_file = os.path.join(res_folder, 'detections_%s_results.json' % self.image_set)
        t0 = time.time()
        self._write_coco_results(detections, res_file)
        self.eval_times = dict(write_s=time.time() - t0)
        if 'test' not in self.image_set:
            info_str, stats = self._do_python_eval(res_file, res_folder)
            return stats

    def coco_results(self, all_boxes):
        """The rows of the results file as columns (image_id, category_id, bbox [N, 4] xywh, score), category-major,
        then image_set_index order, then row order: coco_results_one_category_kernel (lib/dataset/coco.py:21-59)."""
        img, cat, dets = [], [], []
        for cls_ind, cls in enumerate(self.classes):
            if cls == '__background__':
                continue
            for im_ind, index in enumerate(self.image_set_index):
                d = np.asarray(all_boxes[cls_ind][im_ind])
                if len(d) == 0:
                    continue
                dets.append(d.astype(np.float64).reshape(len(d), -1))
                img.append(np.full(len(d), index, np.int64))
                cat.append(np.full(len(d), self._class_to_coco_ind[cls], np.int64))
        if not dets:
            return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 4)), np.zeros(0)
        d = np.concatenate(dets)
        xs, ys = d[:, 0], d[:, 1]
        bbox = round_py2(np.stack([xs, ys, d[:, 2] - xs + 1, d[:, 3] - ys + 1], 1), 1)
        return np.concatenate(img), np.concatenate(cat), bbox, round_py2(d[:, -1], 8)

    def _write_coco_results(self, all_boxes, res_file):
        img, cat, bbox, score = self.coco_results(all_boxes)
        if not (np.isfinite(bbox).all() and np.isfinite(score).all()):
            raise ValueError('evaluate_detections: a detection box or score is not finite')
        print('Writing results json to %s' % res_file)
        fmt = '{"bbox": [%r, %r, %r, %r], "category_id": %d, "image_id": %d, "score": %r}'
        rows = [fmt % (b[0], b[1], b[2], b[3], c, i, s)
                for b, c, i, s in zip(bbox.tolist(), cat.tolist(), img.tolist(), score.tolist())]
        with open(res_file, 'w') as f:
            f.write('[' + ', '.join(rows) + ']')

    def _do_python_eval(self, res_file, res_folder):
        t0 = time.time()
        coco_dt = self.coco.loadRes(res_file)
        coco_eval = COCOeval(self.coco, coco_dt, device=self.device)
        coco_eval.params.useSegm = 0
        t1 = time.time()
        coco_eval.evaluate()
        coco_eval.accumulate()
        torch.cuda.synchronize()
        self.eval_times.update(load_s=t1 - t0, eval_s=time.time() - t1, **coco_eval.times)
        return self._print_detection_metrics(coco_eval)

    def _print_detection_metrics(self, coco_eval):
        """The per-class AP table of lib/dataset/coco.py:338-375 (IoU 0.50:0.95, all areas, 100 detections), then
        COCOeval.summarize()."""
        info_str = ''
        IoU_lo_thresh, IoU_hi_thresh = 0.5, 0.95

        def _get_thr_ind(coco_eval, thr):
            ind = np.where((coco_eval.params.iouThrs > thr - 1e-5) & (coco_eval.params.iouThrs < thr + 1e-5))[0][0]
            assert np.isclose(coco_eval.params.iouThrs[ind], thr)
            return ind

        ind_lo = _get_thr_ind(coco_eval, IoU_lo_thresh)
        ind_hi = _get_thr_ind(coco_eval, IoU_hi_thresh)
        precision = coco_eval.eval['precision'][ind_lo:(ind_hi + 1), :, :, 0, 2]
        ap_default = np.mean(precision[precision > -1])
        line = '~~~~ Mean and per-category AP @ IoU=%.2f,%.2f] ~~~~' % (IoU_lo_thresh, IoU_hi_thresh)
        print(line)
        info_str += line + '\n'
        print('%-15s %5.1f' % ('all', 100 * ap_default))
        info_str += '%-15s %5.1f\n' % ('all', 100 * ap_default)
        for cls_ind, cls in enumerate(self.classes):
            if cls == '__background__':
                continue
            precision = coco_eval.eval['precision'][ind_lo:(ind_hi + 1), :, cls_ind - 1, 0, 2]
            ap = np.mean(precision[precision > -1]) if (precision > -1).any() else float('nan')
            print('%-15s %5.1f' % (cls, 100 * ap))
            info_str += '%-15s %5.1f\n' % (cls, 100 * ap)
        print('~~~~ Summary metrics ~~~~')
        stats = coco_eval.summarize()
        return info_str, stats
