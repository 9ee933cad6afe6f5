"""The `PascalVOC` imdb of the reference (lib/dataset/pascal_voc.py) and its metric, voc_eval
(lib/dataset/pascal_voc_eval.py), with the matching and the AP on the device.

evaluate_detections(all_boxes) writes `results/VOC<year>/Main/comp4_det_<image_set>_<class>.txt` with the reference's
text and scores those files the way do_python_eval does: AP of every class at overlap 0.5, then at 0.7, the 11-point
metric for years before 2010 and the area metric after, and returns the reference's info string.  all_boxes[class][i]
is the [n, 5] (x1, y1, x2, y2, score) array of class `class` in image i of `image_set_index`, gt_roidb's order.

What the device scores is what the files hold: they are parsed back.  The order of the detections is computed on the
host with the reference's own call, np.argsort(-confidence) per class: that sort is not stable, the scores come back
from 3-decimal text and tie often, and the tie order decides which detection takes a GT.  The device takes that order
as input (ops.voc_match / ops.voc_accumulate, csrc/voc_eval.cu) and reproduces the rest in float64 without FMA, the
area metric's np.sum in numpy's pairwise order included, so rec, prec and ap equal the reference's byte for byte.

Differences from the reference: the writer is vectorised; the rows keep Python 2 numpy's arithmetic (coordinates + 1
in float64, whatever the dtype of all_boxes); the annotation cache is this module's own pickle (a Python 2 one at the
same path is read too); and image_set names ('2007_test') give the reference's imdb name, 'PASCALVOC_2007_test'.
"""
import os
import pickle
import time
import xml.etree.ElementTree as ET

import numpy as np
import torch

from . import ops, recall

CLASSES = ('__background__',  # always index 0
           'aeroplane', 'bicycle', 'bird', 'boat', 'bottle', 'bus', 'car', 'cat', 'chair', 'cow', 'diningtable', 'dog',
           'horse', 'motorbike', 'person', 'pottedplant', 'sheep', 'sofa', 'train', 'tvmonitor')
ROW = '{:s} {:.3f} {:.1f} {:.1f} {:.1f} {:.1f}\n'


def parse_voc_rec(filename):
    """One dict per object of a VOC annotation (pascal_voc_eval.py:17-36): name, difficult, bbox as int(float(text))."""
    objects = []
    for obj in ET.parse(filename).findall('object'):
        bbox = obj.find('bndbox')
        objects.append({'name': obj.find('name').text,
                        'difficult': int(obj.find('difficult').text),
                        'bbox': [int(float(bbox.find(k).text)) for k in ('xmin', 'ymin', 'xmax', 'ymax')]})
    return objects


def voc_ap(rec, prec, use_07_metric=False):
    """voc_ap (pascal_voc_eval.py:39-70) on the host: the 11-point metric over np.arange(0., 1.1, 0.1), or the area
    under the precision envelope at the points where the recall changes."""
    rec, prec = np.asarray(rec, np.float64), np.asarray(prec, np.float64)
    if use_07_metric:
        ap = 0.
        for t in np.arange(0., 1.1, 0.1):
            sel = rec >= t
            ap += (0 if not sel.any() else np.max(prec[sel])) / 11.
        return ap
    mrec = np.concatenate(([0.], rec, [1.]))
    mpre = np.maximum.accumulate(np.concatenate(([0.], prec, [0.]))[::-1])[::-1]
    i = np.where(mrec[1:] != mrec[:-1])[0]
    return np.sum((mrec[i + 1] - mrec[i]) * mpre[i + 1])


def _image_names(imageset_file):
    with open(imageset_file, 'r') as f:
        return [x.strip() for x in f.readlines()]


def load_annotations(annopath, image_names, annocache):
    """{image name: parse_voc_rec(...)}, read from annocache when it exists, else parsed and written there."""
    if os.path.isfile(annocache):
        with open(annocache, 'rb') as f:
            return pickle.load(f, encoding='latin1')
    recs = {name: parse_voc_rec(annopath.format(name)) for name in image_names}
    print('saving annotations cache to {:s}'.format(annocache))
    with open(annocache, 'wb') as f:
        pickle.dump(recs, f, pickle.HIGHEST_PROTOCOL)
    return recs


def gt_csr(recs, image_names, classnames):
    """The GTs of voc_eval's class_recs (pascal_voc_eval.py:103-114) for every class as one CSR over the pairs
    p = c * len(image_names) + i: boxes [G, 4] float64, difficult [G] uint8, offsets [P + 1] int32 and npos [C] (the
    non-difficult count of each class).  Objects keep their annotation order; names match exactly."""
    cls_index = {c: k for k, c in enumerate(classnames)}
    key, box, diff = [], [], []
    for i, name in enumerate(image_names):
        for obj in recs[name]:
            k = cls_index.get(obj['name'])
            if k is not None:
                key.append(k * len(image_names) + i)
                box.append(obj['bbox'])
                diff.append(obj['difficult'])
    P = len(classnames) * len(image_names)
    key = np.asarray(key, np.int64)
    order = np.argsort(key, kind='stable')
    off = np.zeros(P + 1, np.int32)
    np.cumsum(np.bincount(key, minlength=P), out=off[1:])
    difficult = np.asarray(diff, bool)[order]
    npos = np.bincount(key[~np.asarray(diff, bool)] // max(len(image_names), 1), minlength=len(classnames))
    return (np.asarray(box, np.float64).reshape(-1, 4)[order], difficult.astype(np.uint8), off,
            npos[:len(classnames)].astype(np.int32))


def read_detections(detfile):
    """The image ids, confidences and boxes of one results file, each number as float() reads it
    (pascal_voc_eval.py:116-124)."""
    with open(detfile, 'r') as f:
        tok = f.read().split()
    a = np.array(tok, dtype=object).reshape(-1, 6)
    return a[:, 0].tolist(), a[:, 1].astype(np.float64), a[:, 2:].astype(np.float64)


def voc_eval_classes(detpath, annopath, imageset_file, classnames, annocache, ovthresh=(0.5,), use_07_metric=False,
                     device="cuda", times=None):
    """voc_eval for several classes and overlap thresholds in one pair of launches.  Returns a dict with, per class,
    sorted_inds (the host's np.argsort(-confidence)), and rec / prec / ap indexed [threshold][class].  times, when a
    dict, gets the seconds spent parsing the files, sorting on the host and on the device (copies included)."""
    t0 = time.time()
    image_names = _image_names(imageset_file)
    recs = load_annotations(annopath, image_names, annocache)
    img_index = {name: i for i, name in enumerate(image_names)}
    gt_box, gt_diff, gt_off, npos = gt_csr(recs, image_names, classnames)
    parsed = []
    for cls in classnames:
        ids, conf, bbox = read_detections(detpath.format(cls))
        parsed.append((np.fromiter((img_index[s] for s in ids), np.int64, len(ids)), conf, bbox))
    t1 = time.time()
    sorted_inds, boxes, pairs = [], [], []
    for c, (img, conf, bbox) in enumerate(parsed):
        # the reference's own call: np.argsort's default kind decides the order of tied scores
        s = np.argsort(-conf) if len(conf) else np.zeros(0, np.int64)
        sorted_inds.append(s)
        boxes.append(bbox[s])
        pairs.append(c * len(image_names) + img[s])
    det_off = np.zeros(len(classnames) + 1, np.int32)
    det_off[1:] = np.cumsum([len(s) for s in sorted_inds])
    t2 = time.time()
    thr = np.asarray(ovthresh, np.float64).reshape(-1)
    dev = torch.device(device)
    flags = ops.voc_match(torch.from_numpy(np.concatenate(boxes).reshape(-1, 4)).to(dev), np.concatenate(pairs),
                          torch.from_numpy(gt_box).to(dev), torch.from_numpy(gt_diff).to(dev), gt_off, thr)
    rec, prec, ap = ops.voc_accumulate(flags, det_off, torch.from_numpy(npos).to(dev), use_07_metric)
    rec, prec, ap = rec.cpu().numpy(), prec.cpu().numpy(), ap.cpu().numpy()
    if times is not None:
        times.update(parse_s=t1 - t0, sort_s=t2 - t1, device_s=time.time() - t2)
    split = lambda a, t: [a[t, det_off[c]:det_off[c + 1]] for c in range(len(classnames))]  # noqa: E731
    return dict(sorted_inds=sorted_inds, rec=[split(rec, t) for t in range(thr.size)],
                prec=[split(prec, t) for t in range(thr.size)], ap=[list(ap[t]) for t in range(thr.size)])


def voc_eval(detpath, annopath, imageset_file, classname, annocache, ovthresh=0.5, use_07_metric=False, device="cuda"):
    """(rec, prec, ap) of one class, as voc_eval (pascal_voc_eval.py:73-181) returns them."""
    r = voc_eval_classes(detpath, annopath, imageset_file, [classname], annocache, (ovthresh,), use_07_metric, device)
    return r['rec'][0][0], r['prec'][0][0], r['ap'][0][0]


def info_string(aps, use_07_metric):
    """do_python_eval's text (pascal_voc.py:417-456) from the APs at 0.5 and 0.7: [(class, ap), ...] each."""
    info_str = 'VOC07 metric? ' + ('Y' if use_07_metric else 'No') + '\n'
    for k, (thr, rows) in enumerate(zip(('0.5', '0.7'), aps)):
        for cls, ap in rows:
            info_str += 'AP for {} = {:.4f}\n'.format(cls, ap)
        info_str += 'Mean AP@{} = {:.4f}'.format(thr, np.mean([ap for _, ap in rows])) + ('\n\n' if k == 0 else '')
    return info_str


class PascalVOC(object):
    def __init__(self, image_set, root_path, devkit_path, result_path=None, device="cuda"):
        """image_set: e.g. 2007_test; root_path: where cache/ goes; devkit_path: holds VOC<year>/ (and results/)."""
        year = image_set.split('_')[0]
        self.image_set = image_set[len(year) + 1:]
        self.name = 'PASCALVOC_' + year + '_' + self.image_set
        self.year = year
        self.root_path, self.devkit_path = root_path, devkit_path
        self.data_path = os.path.join(devkit_path, 'VOC' + year)
        self._result_path = result_path
        self.device = device
        self.classes = list(CLASSES)
        self.num_classes = len(self.classes)
        self.image_set_index = self.load_image_set_index()
        self.num_images = len(self.image_set_index)
        self.config = {'comp_id': 'comp4', 'use_diff': False, 'min_size': 2}
        self.eval_times = {}

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

    def load_image_set_index(self):
        f = os.path.join(self.data_path, 'ImageSets', 'Main', self.image_set + '.txt')
        assert os.path.exists(f), 'Path does not exist: {}'.format(f)
        return _image_names(f)

    def image_path_from_index(self, index):
        image_file = os.path.join(self.data_path, 'JPEGImages', index + '.jpg')
        assert os.path.exists(image_file), 'Path does not exist: {}'.format(image_file)
        return image_file

    def gt_roidb(self):
        """One roidb entry per image (pascal_voc.py:92-109), cached as <name>_gt_roidb.pkl."""
        cache_file = os.path.join(self.cache_path, self.name + '_gt_roidb.pkl')
        if os.path.exists(cache_file):
            with open(cache_file, 'rb') as f:
                roidb = pickle.load(f, encoding='latin1')
            print('{} gt roidb loaded from {}'.format(self.name, cache_file))
            return roidb
        gt_roidb = [self.load_pascal_annotation(index) for index in self.image_set_index]
        with open(cache_file, 'wb') as f:
            pickle.dump(gt_roidb, f, pickle.HIGHEST_PROTOCOL)
        print('wrote gt roidb to {}'.format(cache_file))
        return gt_roidb

    def load_pascal_annotation(self, index):
        """pascal_voc.py:130-178: the non-difficult objects, pixel indexes made 0-based (float(text) - 1) and cast to
        uint16; height and width as floats."""
        tree = ET.parse(os.path.join(self.data_path, 'Annotations', index + '.xml'))
        size = tree.find('size')
        objs = tree.findall('object')
        if not self.config['use_diff']:
            objs = [obj for obj in objs if int(obj.find('difficult').text) == 0]
        class_to_index = dict(zip(self.classes, range(self.num_classes)))
        boxes = np.zeros((len(objs), 4), dtype=np.uint16)
        gt_classes = np.zeros(len(objs), dtype=np.int32)
        overlaps = np.zeros((len(objs), self.num_classes), dtype=np.float32)
        for ix, obj in enumerate(objs):
            bbox = obj.find('bndbox')
            boxes[ix, :] = [float(bbox.find(k).text) - 1 for k in ('xmin', 'ymin', 'xmax', 'ymax')]
            cls = class_to_index[obj.find('name').text.lower().strip()]
            gt_classes[ix] = cls
            overlaps[ix, cls] = 1.0
        return {'image': self.image_path_from_index(index),
                'height': float(size.find('height').text),
                'width': float(size.find('width').text),
                'boxes': boxes,
                'gt_classes': gt_classes,
                'gt_overlaps': overlaps,
                'max_classes': overlaps.argmax(axis=1),
                'max_overlaps': overlaps.max(axis=1),
                'flipped': False}

    def get_result_file_template(self):
        """results/VOC<year>/Main/comp4_det_<image_set>_{:s}.txt under result_path."""
        folder = os.path.join(self.result_path, 'results', 'VOC' + self.year, 'Main')
        return os.path.join(folder, self.config['comp_id'] + '_det_' + self.image_set + '_{:s}.txt')

    def results_text(self, all_boxes, cls_ind):
        """The text write_pascal_results (pascal_voc.py:395-415) writes for one class: '{:s} {:.3f} {:.1f} ...' per
        row, images in image_set_index order, coordinates + 1 added in float64."""
        ids, rows = [], []
        for im_ind, index in enumerate(self.image_set_index):
            dets = all_boxes[cls_ind][im_ind]
            if len(dets) == 0:
                continue
            d = np.asarray(dets)
            rows.append(np.asarray(d, np.float64).reshape(len(d), -1))
            ids += [index] * len(d)
        if not rows:
            return ''
        d = np.concatenate(rows)
        cols = [d[:, -1]] + [d[:, k] + 1 for k in range(4)]
        fmt = ROW.replace('{:s}', '%s').replace('{:.3f}', '%.3f').replace('{:.1f}', '%.1f')
        return ''.join(map(fmt.__mod__, zip(ids, *(c.tolist() for c in cols))))

    def write_pascal_results(self, all_boxes):
        for cls_ind, cls in enumerate(self.classes):
            if cls == '__background__':
                continue
            with open(self.get_result_file_template().format(cls), 'wt') as f:
                f.write(self.results_text(all_boxes, cls_ind))

    def evaluate_recall(self, roidb, candidate_boxes=None, thresholds=None):
        """Proposal recall per GT area range of the first num_images entries of roidb (recall.evaluate_recall): the
        reference's info string, printed and returned."""
        return recall.evaluate_recall(roidb, candidate_boxes, thresholds, num_images=self.num_images,
                                      device=self.device)

    def evaluate_detections(self, detections):
        """Writes the comp4 files and evaluates them (pascal_voc.py:246-265); returns do_python_eval's info string.
        eval_times gets the seconds spent writing, parsing, sorting on the host and on the device."""
        os.makedirs(os.path.join(self.result_path, 'results', 'VOC' + self.year, 'Main'), exist_ok=True)
        t0 = time.time()
        self.write_pascal_results(detections)
        self.eval_times = dict(write_s=time.time() - t0)
        return self.do_python_eval()

    def do_python_eval(self):
        """AP of every class at 0.5 and 0.7 (pascal_voc.py:417-456), both thresholds in one pair of launches."""
        annopath = os.path.join(self.data_path, 'Annotations', '{0!s}.xml')
        imageset_file = os.path.join(self.data_path, 'ImageSets', 'Main', self.image_set + '.txt')
        annocache = os.path.join(self.cache_path, self.name + '_annotations.pkl')
        # the PASCAL VOC metric changed in 2010
        use_07_metric = self.year == 'SDS' or int(self.year) < 2010
        classes = self.classes[1:]
        r = voc_eval_classes(self.get_result_file_template(), annopath, imageset_file, classes, annocache,
                             (0.5, 0.7), use_07_metric, self.device, self.eval_times)
        info_str = info_string([list(zip(classes, r['ap'][0])), list(zip(classes, r['ap'][1]))], use_07_metric)
        print(info_str)
        return info_str
