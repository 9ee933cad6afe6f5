"""TEST INFRASTRUCTURE ONLY.  Runs the reference's OWN PASCAL VOC evaluation in THIS container and writes
tests/golden/voc_eval_ref.npz (run: python oracle/run_ref_voc_eval.py):

  parse_voc_rec, voc_ap, voc_eval          lib/dataset/pascal_voc_eval.py
  PascalVOC (load_pascal_annotation,       lib/dataset/pascal_voc.py, on the IMDB base class of lib/dataset/imdb.py
  write_pascal_results, do_python_eval)

The sources are read as text from /root/reference and executed in memory (nothing is copied into the repo).  They are
Python 2, so Python-2-only tokens are rewritten: print statements, cPickle, xrange, np.bool; the imports the evaluation
does not reach (cv2, PIL, mask, bbox, nms, ds_utils, multiprocessing) are dropped.  The arithmetic and the control flow
are the reference's.  np.argsort is wrapped to record the order voc_eval computes (sorted_inds).

all_boxes holds float32 values passed as float64: the reference's `dets[k, 0] + 1` ran under Python 2 numpy, whose
scalar promotion made it a float64 sum; under numpy 2 a float32 row would add in float32.

Every case is a synthetic VOCdevkit written to a temporary directory: XML annotations, an image set, empty JPEG files,
and all_boxes.  Per case the fixture records the inputs, the comp4 file text, gt_roidb, and for every class, overlap
threshold (0.5, 0.7) and metric (11-point, area) voc_eval's sorted_inds, rec, prec and ap, plus do_python_eval's
info_str for the case's year."""
import os
import re
import sys
import tempfile
import types

import numpy as np

REF = "/root/reference/lib/dataset"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "tests", "golden", "voc_eval_ref.npz")
CLASSES = ['aeroplane', 'bicycle', 'bird', 'boat', 'bottle', 'bus', 'car', 'cat', 'chair', 'cow', 'diningtable', 'dog',
           'horse', 'motorbike', 'person', 'pottedplant', 'sheep', 'sofa', 'train', 'tvmonitor']
DROP = ('import cv2', 'import PIL', 'from PIL import Image', 'from mask.mask_transform import',
        'from bbox.bbox_transform import', 'from nms.nms import', 'from multiprocessing import', 'from ds_utils import',
        'from imdb import IMDB', 'from pascal_voc_eval import')


def _py3(src):
    src = '\n'.join('' if l.strip().startswith(DROP) else l for l in src.split('\n'))
    src = re.sub(r'^(\s*)print (.+)$', r'\1print(\2)', src, flags=re.M)
    src = src.replace('import cPickle', 'import pickle as cPickle').replace('xrange(', 'range(')
    src = re.sub(r'\bnp\.bool\b', 'bool', src)
    return src


class _RecordingNumpy(types.ModuleType):
    """numpy, with every argsort result kept in `calls`."""
    def __init__(self):
        super().__init__("numpy")
        self.calls = []

    def __getattr__(self, k):
        return getattr(np, k)

    def argsort(self, *a, **kw):
        r = np.argsort(*a, **kw)
        self.calls.append(r)
        return r


def load_reference():
    """(PascalVOC class, voc_eval namespace) of the reference."""
    ev = {"__name__": "ref_pascal_voc_eval"}
    exec(compile(_py3(open(os.path.join(REF, "pascal_voc_eval.py")).read()), "pascal_voc_eval.py", "exec"), ev)
    ev["np"] = _RecordingNumpy()
    im = {"__name__": "ref_imdb"}
    exec(compile(_py3(open(os.path.join(REF, "imdb.py")).read()), "imdb.py", "exec"), im)
    pv = {"__name__": "ref_pascal_voc", "IMDB": im["IMDB"], "voc_eval": ev["voc_eval"], "voc_eval_sds": None}
    exec(compile(_py3(open(os.path.join(REF, "pascal_voc.py")).read()), "pascal_voc.py", "exec"), pv)
    return pv["PascalVOC"], ev


# --------------------------------------------------------------------------------------------------------------------
# cases: objects are (name, difficult, xmin, ymin, xmax, ymax) in XML text; detections (class index 1..20, image,
# x1, y1, x2, y2, score) in all_boxes coordinates (0-based: the file holds them + 1)
# --------------------------------------------------------------------------------------------------------------------
def case_hand():
    """Hand-made edge cases, year 2012 (the area metric's NaN reaches the info string)."""
    images = ['000001', '000002', '000003', '000004', '000005']
    objs = {
        # aeroplane: GT 1..10 x 1..10 (area 100)
        '000001': [('aeroplane', 0, '1', '1', '10', '10'), ('aeroplane', 0, '31', '31', '40', '40'),
                   ('aeroplane', 0, '31', '31', '40', '40'),  # two identical GTs: equal IoUs, first argmax
                   ('bicycle', 1, '1', '1', '20', '20'),       # difficult
                   ('bicycle', 0, '50', '50', '80.7', '90.2'),
                   ('bird', 1, '5', '5', '25', '25')],          # bird: all GTs difficult (npos = 0)
        '000002': [('bird', 1, '10', '10', '30', '30'), ('cat', 0, '2', '3', '40', '50'),
                   ('cat', 0, '100', '100', '150', '140')],
        '000003': [],                                          # no objects
        '000004': [('person', 0, '10', '10', '60', '110'), ('person', 0, '70', '10', '120', '110'),
                   ('person', 0, '130', '10', '180', '110'), ('person', 1, '200', '10', '250', '110')],
        '000005': [('boat', 0, '1', '1', '50', '50')],
    }
    d = []
    # aeroplane: IoU exactly 0.5 (strict compare: an fp at 0.5), a hit, a duplicate, the tied pair
    d += [(1, 0, 0, 0, 9, 4, 0.9), (1, 0, 0, 0, 9, 9, 0.8), (1, 0, 0, 0, 9, 9, 0.8), (1, 0, 30, 30, 39, 39, 0.7),
          (1, 0, 30, 30, 39, 39, 0.7), (1, 0, 30, 30, 39, 39, 0.7), (1, 2, 0, 0, 9, 9, 0.95)]
    # bicycle: on the difficult GT (neither tp nor fp), then the real one, a zero-width detection
    d += [(2, 0, 0, 0, 19, 19, 0.99), (2, 0, 49, 49, 79.7, 89.2, 0.5), (2, 0, 49, 49, 48, 89, 0.6)]
    # bird: detections on the difficult-only class
    d += [(3, 0, 4, 4, 24, 24, 0.9), (3, 1, 9, 9, 29, 29, 0.3), (3, 3, 0, 0, 5, 5, 0.1)]
    # cat: scores that round to a tie in 3 decimals
    d += [(8, 1, 1, 2, 39, 49, 0.50049), (8, 1, 99, 99, 149, 139, 0.5004), (8, 1, 1, 2, 39, 49, 0.50041),
          (8, 2, 1, 1, 9, 9, 0.5001)]
    # person: three at each GT with equal scores, one on the difficult GT, rounding at .x5 in coordinates
    for k, x in enumerate((9, 69, 129, 199)):
        d += [(15, 3, x + 0.25, 9.05, x + 50.75, 109.15, 0.25), (15, 3, x + 2, 12, x + 40, 100, 0.25)]
    # boat: no detections
    return '2012', images, objs, d


def case_seeded(seed, year, n_img, per_img, n_det, score_decimals, heavy_class=None):
    rng = np.random.RandomState(seed)
    images = ['%06d' % (7 * i + 3) for i in range(n_img)]
    objs, d = {}, []
    for i, name in enumerate(images):
        W, H = rng.randint(200, 500), rng.randint(200, 500)
        o = []
        for _ in range(rng.poisson(per_img)):
            c = heavy_class if heavy_class is not None and rng.rand() < 0.6 else rng.randint(20)
            w, h = rng.randint(8, W // 2), rng.randint(8, H // 2)
            x, y = rng.randint(1, W - w), rng.randint(1, H - h)
            o.append((CLASSES[c], int(rng.rand() < 0.15), str(x), str(y), str(x + w), str(y + h)))
        objs[name] = o
        for _ in range(n_det):
            if o and rng.rand() < 0.7:
                g = o[rng.randint(len(o))]
                c = CLASSES.index(g[0]) if rng.rand() < 0.85 else rng.randint(20)
                b = np.array([float(v) for v in g[2:]]) - 1
                b += rng.randn(4) * rng.choice([0.5, 3.0, 12.0])
            else:
                c = rng.randint(20)
                b = np.array([rng.uniform(0, W - 20), rng.uniform(0, H - 20), 0, 0])
                b[2:] = b[:2] + rng.uniform(2, 150, 2)
            b = np.round(b * 4) / 4 if rng.rand() < 0.3 else b   # exact .x5 values in the file
            d.append((c + 1, i) + tuple(b) + (round(rng.rand(), score_decimals),))
    return year, images, objs, d


CASES = {
    "hand": case_hand,
    "ties07": lambda: case_seeded(1, '2007', 80, 4, 12, 2),
    "ties12": lambda: case_seeded(2, '2012', 120, 5, 10, 2, heavy_class=14),
}


def xml_text(objs, W=500, H=375):
    o = ''.join('<object><name>%s</name><difficult>%d</difficult><bndbox><xmin>%s</xmin><ymin>%s</ymin>'
                '<xmax>%s</xmax><ymax>%s</ymax></bndbox></object>' % ob for ob in objs)
    return '<annotation><size><width>%d</width><height>%d</height></size>%s</annotation>' % (W, H, o)


def write_devkit(root, year, images, objs):
    dk = os.path.join(root, 'VOCdevkit')
    vp = os.path.join(dk, 'VOC' + year)
    for sub in ('Annotations', 'ImageSets/Main', 'JPEGImages'):
        os.makedirs(os.path.join(vp, sub), exist_ok=True)
    with open(os.path.join(vp, 'ImageSets', 'Main', 'test.txt'), 'w') as f:
        f.write(''.join(n + '\n' for n in images))
    for n in images:
        with open(os.path.join(vp, 'Annotations', n + '.xml'), 'w') as f:
            f.write(xml_text(objs[n]))
        open(os.path.join(vp, 'JPEGImages', n + '.jpg'), 'w').close()
    return dk


def all_boxes_of(d, n_img):
    """float32 rows as float64 (see the module docstring), [21][n_img] lists."""
    ab = [[np.zeros((0, 5), np.float64) for _ in range(n_img)] for _ in range(21)]
    rows = {}
    for c, i, *v in d:
        rows.setdefault((c, i), []).append(v)
    for (c, i), v in rows.items():
        ab[c][i] = np.asarray(v, np.float32).astype(np.float64)
    return ab


def run_case(PascalVOC, ev, name, out):
    year, images, objs, d = CASES[name]()
    with tempfile.TemporaryDirectory() as root:
        dk = write_devkit(root, year, images, objs)
        imdb = PascalVOC(year + '_test', root, dk)
        roidb = imdb.gt_roidb()
        ab = all_boxes_of(d, len(images))
        os.makedirs(os.path.join(imdb.result_path, 'results', 'VOC' + year, 'Main'), exist_ok=True)
        info = imdb.evaluate_detections(ab)
        tmpl = imdb.get_result_file_template()
        texts = [open(tmpl.format(c)).read() for c in CLASSES]
        annopath = os.path.join(imdb.data_path, 'Annotations', '{0!s}.xml')
        imageset = os.path.join(imdb.data_path, 'ImageSets', 'Main', 'test.txt')
        cache = os.path.join(imdb.cache_path, imdb.name + '_annotations.pkl')
        for metric in ('07', 'area'):
            for thr in ('0.5', '0.7'):
                inds, rec, prec, ap = [], [], [], []
                for c in CLASSES:
                    ev['np'].calls.clear()
                    r, p, a = ev['voc_eval'](tmpl.format(c), annopath, imageset, c, cache, ovthresh=float(thr),
                                             use_07_metric=metric == '07')
                    inds.append(ev['np'].calls[0] if ev['np'].calls else np.zeros(0, np.int64))
                    rec.append(r)
                    prec.append(p)
                    ap.append(a)
                k = '%s_%s_%s_' % (name, metric, thr)
                out[k + 'rec'] = np.concatenate(rec).astype(np.float64)
                out[k + 'prec'] = np.concatenate(prec).astype(np.float64)
                out[k + 'ap'] = np.asarray(ap, np.float64)
                si = np.concatenate(inds).astype(np.int64)
                if name + '_sorted_inds' in out:
                    assert out[name + '_sorted_inds'].tobytes() == si.tobytes()
                out[name + '_sorted_inds'] = si
                out[name + '_det_off'] = np.concatenate([[0], np.cumsum([len(x) for x in inds])]).astype(np.int64)
    out[name + '_year'] = np.array(year)
    out[name + '_images'] = np.array(images)
    out[name + '_xml'] = np.array([xml_text(objs[n]) for n in images])
    out[name + '_dets'] = np.array([[c, i] + list(v) for c, i, *v in d], np.float64).reshape(-1, 7)
    out[name + '_text'] = np.array(texts)
    out[name + '_info'] = np.array(info)
    n = [len(r['boxes']) for r in roidb]
    out[name + '_roidb_n'] = np.asarray(n, np.int64)
    out[name + '_roidb_hw'] = np.array([[r['height'], r['width']] for r in roidb], np.float64)
    for k in ('boxes', 'gt_classes', 'gt_overlaps', 'max_classes', 'max_overlaps'):
        out[name + '_roidb_' + k] = np.concatenate([r[k] for r in roidb])
    out[name + '_roidb_flipped'] = np.array([r['flipped'] for r in roidb])
    out[name + '_roidb_image'] = np.array([os.path.relpath(r['image'], dk) for r in roidb])


def main():
    PascalVOC, ev = load_reference()
    out = {}
    for name in CASES:
        run_case(PascalVOC, ev, name, out)
        print(name, 'detections', len(out[name + '_sorted_inds']))
    np.savez_compressed(OUT, **out)
    print('wrote', os.path.relpath(OUT), os.path.getsize(OUT), 'bytes')


if __name__ == "__main__":
    sys.exit(main())
