"""COCO box evaluation: the `COCO`, `COCOeval` and `Params` of the reference's pycocotools
(lib/dataset/pycocotools/coco.py, cocoeval.py), with the per-image matching and the accumulation on the device.

    reference                                              here
    computeIoU -> mask.iou -> bbIou (maskApi.c)            `sniper_coco_box_iou_batched` (COCOeval.ious, on request)
    evaluateImg, per (image, category, area) in Python     `sniper_coco_match`: every pair x area x IoU threshold,
                                                           one launch
    accumulate, per (category, area, maxDet) in Python     one stable device sort per category + `sniper_coco_accumulate`
    summarize                                              the same numpy expressions on the device's arrays

`precision`, `recall` and `stats` equal the reference's byte for byte: every operation involved is an IEEE double add,
multiply, divide, min, max or compare, done in the reference's order.  `evalImgs` (1.6 M dicts on val2017, what makes
the reference slow) is built only when it is read.  Box evaluation only: `useSegm=1` (no mask branch here) and
`useCats=0` (SNIPER never evaluates without categories) are refused.
"""
import copy
import datetime
import itertools
import json
import numbers
import time
from collections import defaultdict

import numpy as np
import torch

from . import ops


def _as_list(v):
    return v if isinstance(v, list) else [v]


class COCO(object):
    """Annotation index of pycocotools' COCO (coco.py:61-328): the accessors the evaluation and the COCO imdb use."""

    def __init__(self, annotation_file=None):
        self.dataset, self.anns, self.imgToAnns, self.catToImgs, self.imgs, self.cats = {}, {}, {}, {}, {}, {}
        self._cols = None
        if annotation_file is not None:
            if isinstance(annotation_file, dict):
                self.dataset = annotation_file
            else:
                with open(annotation_file, 'r') as f:
                    self.dataset = json.load(f)
            self.createIndex()

    def createIndex(self):
        anns, imgs, cats = {}, {}, {}
        imgToAnns, catToImgs = defaultdict(list), defaultdict(list)
        for ann in self.dataset.get('annotations', []):
            imgToAnns[ann['image_id']].append(ann)
            anns[ann['id']] = ann
        for img in self.dataset.get('images', []):
            imgs[img['id']] = img
        for cat in self.dataset.get('categories', []):
            cats[cat['id']] = cat
        if 'annotations' in self.dataset and 'categories' in self.dataset:
            catToImgs = {cat['id']: [] for cat in self.dataset['categories']}
            for ann in self.dataset['annotations']:
                catToImgs[ann['category_id']].append(ann['image_id'])
        self.anns, self.imgToAnns, self.catToImgs, self.imgs, self.cats = anns, dict(imgToAnns), catToImgs, imgs, cats
        self._cols = None

    def getAnnIds(self, imgIds=[], catIds=[], areaRng=[], iscrowd=None):
        imgIds, catIds = _as_list(imgIds), _as_list(catIds)
        if len(imgIds) == len(catIds) == len(areaRng) == 0:
            anns = self.dataset['annotations']
        else:
            if len(imgIds):
                anns = list(itertools.chain.from_iterable(self.imgToAnns[i] for i in imgIds if i in self.imgToAnns))
            else:
                anns = self.dataset['annotations']
            anns = anns if len(catIds) == 0 else [a for a in anns if a['category_id'] in catIds]
            anns = anns if len(areaRng) == 0 else [a for a in anns if areaRng[0] < a['area'] < areaRng[1]]
        if iscrowd is not None:
            return [a['id'] for a in anns if a['iscrowd'] == iscrowd]
        return [a['id'] for a in anns]

    def getCatIds(self, catNms=[], supNms=[], catIds=[]):
        catNms, supNms, catIds = _as_list(catNms), _as_list(supNms), _as_list(catIds)
        cats = self.dataset['categories']
        cats = cats if len(catNms) == 0 else [c for c in cats if c['name'] in catNms]
        cats = cats if len(supNms) == 0 else [c for c in cats if c['supercategory'] in supNms]
        cats = cats if len(catIds) == 0 else [c for c in cats if c['id'] in catIds]
        return [c['id'] for c in cats]

    def getImgIds(self, imgIds=[], catIds=[]):
        imgIds, catIds = _as_list(imgIds), _as_list(catIds)
        if len(imgIds) == len(catIds) == 0:
            return list(self.imgs.keys())
        ids = set(imgIds)
        for i, catId in enumerate(catIds):
            if i == 0 and len(ids) == 0:
                ids = set(self.catToImgs[catId])
            else:
                ids &= set(self.catToImgs[catId])
        return list(ids)

    @staticmethod
    def _load(table, ids):
        if isinstance(ids, numbers.Integral):
            return [table[ids]]
        return [table[i] for i in ids]

    def loadAnns(self, ids=[]):
        return self._load(self.anns, ids)

    def loadCats(self, ids=[]):
        return self._load(self.cats, ids)

    def loadImgs(self, ids=[]):
        return self._load(self.imgs, ids)

    def loadRes(self, resFile):
        """Result api object of a box results file (a path or the parsed list), as coco.py:282-328: area = w * h,
        id = position + 1, iscrowd = 0.  Every result's image must be in this set."""
        res = COCO()
        res.dataset['images'] = [img for img in self.dataset['images']]
        if isinstance(resFile, str):
            with open(resFile) as f:
                anns = json.load(f)
        else:
            anns = resFile
        if not isinstance(anns, list):
            raise TypeError('results in not an array of objects')
        if len(anns) == 0:
            raise ValueError('loadRes: the results list is empty (nothing to evaluate)')
        annsImgIds = set(a['image_id'] for a in anns)
        assert annsImgIds == (annsImgIds & set(self.getImgIds())), 'Results do not correspond to current coco set'
        if 'bbox' not in anns[0] or anns[0]['bbox'] == []:
            raise ValueError('loadRes: only box results are supported (no segmentation or caption results)')
        res.dataset['categories'] = copy.deepcopy(self.dataset['categories'])
        bb = np.array([a['bbox'] for a in anns], dtype=np.float64).reshape(-1, 4)
        area = (bb[:, 2] * bb[:, 3]).tolist()
        for i, a in enumerate(anns):
            a['area'] = area[i]
            a['id'] = i + 1
            a['iscrowd'] = 0
        res.dataset['annotations'] = anns
        res.createIndex()
        return res

    def columns(self):
        """The annotations as numpy columns in list order (cached): image_id, category_id, bbox [N, 4], area,
        iscrowd, ignore, id, score (NaN where absent)."""
        if self._cols is None:
            anns = self.dataset.get('annotations', [])
            self._cols = dict(
                image_id=np.array([a['image_id'] for a in anns], dtype=np.int64),
                category_id=np.array([a['category_id'] for a in anns], dtype=np.int64),
                bbox=np.array([a['bbox'] for a in anns], dtype=np.float64).reshape(-1, 4),
                area=np.array([a['area'] for a in anns], dtype=np.float64),
                iscrowd=np.array([a['iscrowd'] for a in anns], dtype=np.int64),
                ignore=np.array([bool(a.get('ignore', 0)) for a in anns], dtype=bool),
                id=np.array([a['id'] for a in anns], dtype=np.int64),
                score=np.array([a.get('score', np.nan) for a in anns], dtype=np.float64))
        return self._cols


class Params(object):
    """Evaluation parameters of cocoeval.py:432-445.  np.linspace gets an integer count (numpy 2 refuses the float the
    reference passes): the same doubles, e.g. 0.8999999999999999 for the ninth IoU threshold."""

    def __init__(self):
        self.imgIds = []
        self.catIds = []
        self.iouThrs = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
        self.recThrs = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
        self.maxDets = [1, 10, 100]
        self.areaRng = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
        self.useSegm = 0
        self.useCats = 1


def pack(cocoGt, cocoDt, p):
    """The CSR the kernels read, from the annotation columns (vectorised): the non-empty (category, image) pairs in
    category-major, params.imgIds order; per pair the GT rows in annotation order (cocoeval's _gts grouping) and the
    detection rows sorted by descending score, stable (its sorted(dt, key=-score)), cut to maxDets[-1]."""
    imgIds = np.asarray(p.imgIds, dtype=np.int64)
    catIds = np.asarray(p.catIds, dtype=np.int64)
    I, K = imgIds.size, catIds.size

    def keys(c):
        """pair key (category index * I + image index) of every row, and whether the row is in the evaluated set"""
        if I == 0 or K == 0:
            return np.zeros(c['id'].shape, np.int64), np.zeros(c['id'].shape, bool)
        ii = np.searchsorted(imgIds, c['image_id']).clip(0, I - 1)
        kk = np.searchsorted(catIds, c['category_id']).clip(0, K - 1)
        ok = (imgIds[ii] == c['image_id']) & (catIds[kk] == c['category_id'])
        return kk.astype(np.int64) * I + ii, ok

    g, d = cocoGt.columns(), cocoDt.columns()
    if np.any((g['iscrowd'] != 0) & (g['iscrowd'] != 1)):
        raise ValueError("pack: iscrowd must be 0 or 1")
    gkey, gok = keys(g)
    gsel = np.flatnonzero(gok)
    gsel = gsel[np.argsort(gkey[gsel], kind='stable')]
    gkey = gkey[gsel]
    dkey, dok = keys(d)
    dsel = np.flatnonzero(dok)
    if np.isnan(d['score'][dsel]).any():
        raise ValueError("pack: a detection has no score or a NaN score")
    dsel = dsel[np.lexsort((-d['score'][dsel], dkey[dsel]))]
    dkey = dkey[dsel]
    rank = np.arange(dkey.size) - np.searchsorted(dkey, dkey, 'left')
    cut = rank < p.maxDets[-1]
    dsel, dkey, rank = dsel[cut], dkey[cut], rank[cut]
    pairs = np.union1d(np.unique(gkey), np.unique(dkey))
    P = pairs.size
    gt_off = np.searchsorted(gkey, np.append(pairs, np.iinfo(np.int64).max), 'left').astype(np.int32)
    dt_off = np.searchsorted(dkey, np.append(pairs, np.iinfo(np.int64).max), 'left').astype(np.int32)
    pair_cat = pairs // max(I, 1)
    return dict(
        I=I, K=K, P=P, pairs=pairs, pair_cat=pair_cat, pair_img=pairs % max(I, 1),
        cat_pair_off=np.searchsorted(pair_cat, np.arange(K + 1), 'left').astype(np.int32),
        gt_off=gt_off, dt_off=dt_off,
        gt_rows=gsel, gt_box=np.ascontiguousarray(g['bbox'][gsel]), gt_area=g['area'][gsel],
        gt_flags=((g['iscrowd'][gsel] == 1) | (g['ignore'][gsel].astype(np.int64) << 1)).astype(np.uint8),
        gt_id=g['id'][gsel],
        dt_rows=dsel, dt_box=np.ascontiguousarray(d['bbox'][dsel]), dt_area=d['area'][dsel], dt_id=d['id'][dsel],
        dt_score=d['score'][dsel], dt_rank=rank.astype(np.int32),
        dt_cat=np.repeat(pair_cat, np.diff(dt_off)).astype(np.int64))


class COCOeval(object):
    """pycocotools' COCOeval for boxes (cocoeval.py:10-430): params, evaluate(), accumulate(), summarize(), stats,
    eval['precision' | 'recall' | 'counts'], and, built when read, ious and evalImgs."""

    def __init__(self, cocoGt=None, cocoDt=None, device="cuda"):
        self.cocoGt, self.cocoDt, self.device = cocoGt, cocoDt, device
        self.params = Params()
        self.eval = {}
        self._paramsEval = {}
        self.stats = []
        self._pk = self._dev = self._match = None
        self._ious = self._evalImgs = None
        self.times = {}
        if cocoGt is not None:
            self.params.imgIds = sorted(cocoGt.getImgIds())
            self.params.catIds = sorted(cocoGt.getCatIds())

    def _to_dev(self, a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(self.device)

    def evaluate(self):
        """Matches every (image, category) pair at every area range and IoU threshold on the device."""
        tic = time.time()
        print('Running per image evaluation...      ')
        p = self.params
        if p.useSegm:
            raise NotImplementedError('COCOeval: segmentation evaluation (useSegm=1) is not supported; set useSegm = 0')
        if not p.useCats:
            raise NotImplementedError('COCOeval: useCats=0 (category-agnostic evaluation) is not supported')
        p.imgIds = list(np.unique(p.imgIds))
        p.catIds = list(np.unique(p.catIds))
        p.maxDets = sorted(p.maxDets)
        self.params = p
        self._pk = pk = pack(self.cocoGt, self.cocoDt, p)
        t1 = time.time()
        self._dev = {k: self._to_dev(pk[k]) for k in ('gt_box', 'gt_area', 'gt_flags', 'gt_id', 'dt_box', 'dt_area',
                                                      'dt_id', 'dt_score', 'dt_rank', 'dt_cat')}
        self._match = self._run_match(full=False)
        torch.cuda.synchronize()
        self.times = dict(pack_s=t1 - tic, match_s=time.time() - t1)
        self._ious = self._evalImgs = None
        self.eval = {}
        self._paramsEval = copy.deepcopy(self.params)
        print('DONE (t=%0.2fs).' % (time.time() - tic))

    def _run_match(self, full):
        pk, dv, p = self._pk, self._dev, self.params
        return ops.coco_match(dv['dt_box'], dv['dt_area'], dv['dt_id'], dv['gt_box'], dv['gt_area'], dv['gt_flags'],
                              dv['gt_id'], pk['dt_off'], pk['gt_off'], np.asarray(p.iouThrs, np.float64),
                              np.asarray(p.areaRng, np.float64), full=full)

    def _pair_lists(self):
        """(image ids, category ids) of the pairs."""
        pk, p = self._pk, self._paramsEval
        return np.asarray(p.imgIds)[pk['pair_img']], np.asarray(p.catIds)[pk['pair_cat']]

    @property
    def ious(self):
        """{(imgId, catId): [D, G] IoU matrix of the score-sorted, maxDets[-1]-cut detections against the GTs, or []}."""
        if self._ious is None:
            if self._pk is None:
                return {}
            pk, p = self._pk, self._paramsEval
            out, off = ops.coco_box_iou_batched(self._dev['dt_box'], self._dev['gt_box'], self._dev['gt_flags'],
                                                pk['dt_off'], pk['gt_off'])
            flat = out.cpu().numpy()
            ious = {(i, c): [] for c in p.catIds for i in p.imgIds}
            nd, ng = np.diff(pk['dt_off']), np.diff(pk['gt_off'])
            img, cat = self._pair_lists()
            for q in range(pk['P']):
                if nd[q] and ng[q]:
                    ious[img[q], cat[q]] = flat[off[q]:off[q + 1]].reshape(nd[q], ng[q])
            self._ious = ious
        return self._ious

    @property
    def evalImgs(self):
        """cocoeval's per (category, area range, image) list of result dicts (None for empty pairs); built on first
        read from a second matching launch that also returns the matched ids and the GT order."""
        if self._evalImgs is None:
            if self._pk is None:
                return []
            pk, p = self._pk, self._paramsEval
            r = {k: v.cpu().numpy() for k, v in self._run_match(full=True).items()}
            I, A, T = pk['I'], len(p.areaRng), len(p.iouThrs)
            out = [None] * (len(p.catIds) * A * I)
            img, cat = self._pair_lists()
            for q in range(pk['P']):
                g0, g1, d0, d1 = pk['gt_off'][q], pk['gt_off'][q + 1], pk['dt_off'][q], pk['dt_off'][q + 1]
                dtIds = pk['dt_id'][d0:d1].tolist()
                dtScores = pk['dt_score'][d0:d1].tolist()
                for a in range(A):
                    order = r['gt_order'][a, g0:g1]
                    gflags, garea = pk['gt_flags'][g0:g1][order], pk['gt_area'][g0:g1][order]
                    lo, hi = p.areaRng[a]
                    gtIg = ((gflags & 3 != 0) | (garea < lo) | (garea > hi)).astype(np.int64)
                    out[(pk['pair_cat'][q] * A + a) * I + pk['pair_img'][q]] = {
                        'image_id': img[q], 'category_id': cat[q], 'aRng': p.areaRng[a], 'maxDet': p.maxDets[-1],
                        'dtIds': dtIds, 'gtIds': pk['gt_id'][g0:g1][order].tolist(),
                        'dtMatches': r['dt_match'][a, :, d0:d1].astype(np.float64),
                        'gtMatches': r['gt_match'][a, :, g0:g1].astype(np.float64),
                        'dtScores': dtScores, 'gtIgnore': gtIg,
                        'dtIgnore': (r['dt_flags'][a, :, d0:d1] & 2) != 0}
            self._evalImgs = out
        return self._evalImgs

    def accumulate(self, p=None):
        """precision [T, R, K, A, M] and recall [T, K, A, M] (-1 where there is no GT) on the device.  Accumulates the
        evaluated setting; a params object whose categories, images, areas or maxDets differ from it is refused."""
        print('Accumulating evaluation results...   ')
        tic = time.time()
        if self._pk is None:
            raise RuntimeError('Please run evaluate() first')
        if p is None:
            p = self.params
        pe = self._paramsEval
        for f in ('imgIds', 'catIds', 'maxDets'):
            if list(getattr(p, f)) != list(getattr(pe, f)):
                raise NotImplementedError('accumulate: params.%s differs from the evaluated one' % f)
        if np.asarray(p.areaRng, np.float64).tobytes() != np.asarray(pe.areaRng, np.float64).tobytes() or \
                np.asarray(p.iouThrs).tobytes() != np.asarray(pe.iouThrs).tobytes():
            raise NotImplementedError('accumulate: params.areaRng / iouThrs differ from the evaluated ones')
        pk, dv, m = self._pk, self._dev, self._match
        cat_order = ops.coco_category_order(dv['dt_score'], dv['dt_cat'])
        precision, recall = ops.coco_accumulate(m['dt_flags'], dv['dt_rank'], cat_order, pk['dt_off'], m['npig'],
                                                pk['cat_pair_off'], p.maxDets, np.asarray(p.recThrs, np.float64))
        T, R, K, A, M = precision.shape
        self.eval = {
            'params': p,
            'counts': [T, R, K, A, M],
            'date': datetime.datetime.now().strftime("%Y-%m-%d %H:%M:%S"),
            'precision': precision.cpu().numpy(),
            'recall': recall.cpu().numpy(),
        }
        self.times['accumulate_s'] = time.time() - tic
        print('DONE (t=%0.2fs).' % (time.time() - tic))

    def summarize(self):
        """The twelve AP / AR lines of cocoeval.py:376-427, same expressions, same printed text."""
        def _summarize(ap=1, iouThr=None, areaRng='all', maxDets=100):
            p = self.params
            iStr = ' {:<18} {} @[ IoU={:<9} | area={:>6} | maxDets={:>3} ] = {}'
            titleStr = 'Average Precision' if ap == 1 else 'Average Recall'
            typeStr = '(AP)' if ap == 1 else '(AR)'
            iouStr = '%0.2f:%0.2f' % (p.iouThrs[0], p.iouThrs[-1]) if iouThr is None else '%0.2f' % (iouThr)
            aind = [i for i, aRng in enumerate(['all', 'small', 'medium', 'large']) if aRng == areaRng]
            mind = [i for i, mDet in enumerate([1, 10, 100]) if mDet == maxDets]
            if ap == 1:
                s = self.eval['precision']
                if iouThr is not None:
                    t = np.where(iouThr == p.iouThrs)[0]
                    s = s[t]
                s = s[:, :, :, aind, mind]
            else:
                s = self.eval['recall']
                s = s[:, :, aind, mind]
            if len(s[s > -1]) == 0:
                mean_s = -1
            else:
                mean_s = np.mean(s[s > -1])
            print(iStr.format(titleStr, typeStr, iouStr, areaRng, '%d' % (maxDets), '%.3f' % (float(mean_s))))
            return mean_s

        if not self.eval:
            raise Exception('Please run accumulate() first')
        self.stats = np.zeros((12,))
        self.stats[0] = _summarize(1)
        self.stats[1] = _summarize(1, iouThr=.5)
        self.stats[2] = _summarize(1, iouThr=.75)
        self.stats[3] = _summarize(1, areaRng='small')
        self.stats[4] = _summarize(1, areaRng='medium')
        self.stats[5] = _summarize(1, areaRng='large')
        self.stats[6] = _summarize(0, maxDets=1)
        self.stats[7] = _summarize(0, maxDets=10)
        self.stats[8] = _summarize(0, maxDets=100)
        self.stats[9] = _summarize(0, areaRng='small')
        self.stats[10] = _summarize(0, areaRng='medium')
        self.stats[11] = _summarize(0, areaRng='large')
        return self.stats
