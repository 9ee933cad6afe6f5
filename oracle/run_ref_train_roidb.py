"""TEST INFRASTRUCTURE ONLY.  Runs the reference's OWN training-roidb code in THIS container and writes
tests/golden/train_roidb_ref.npz (run: python oracle/run_ref_train_roidb.py, after build_ref_cython.py):

  load_proposal_roidb, merge_roidb,        lib/data_utils/load_data.py
  filter_roidb
  append_flipped_images, rpn_roidb,        lib/dataset/imdb.py (the IMDB base of PascalVOC), with the reference's Cython
  create_roidb_from_box_list, merge_roidbs bbox_overlaps (oracle/_ref/ref_bbox)
  PascalVOC.gt_roidb                       lib/dataset/pascal_voc.py
  add_bbox_regression_targets              lib/bbox/bbox_regression.py over lib/bbox/bbox_transform.py

in main_train.py's order (:54-66) on a synthetic VOCdevkit (2007_trainval + 2012_trainval) written to a temporary
directory, for both branches of load_proposal_roidb: only_gt, and rpn with the NMS-ed proposals in the
`<name>_rpn_after_nms.pkl` cache (the file load_rpn_data reads before it would run its NMS).  Every branch runs with
precomputed and accumulated normalisation, class-agnostic and per-class.

The sources are read as text from /root/reference and executed in memory (nothing is copied into the repo), with the
Python-2-only tokens rewritten as oracle/run_ref_voc_eval.py does, plus np.float -> float (and comments after a
print statement dropped).  The arithmetic and the
control flow are the reference's.  The fixture holds the devkit (XML text, image lists), the proposals and, per case,
the final roidb: entry order (image, flipped), the row arrays concatenated with per-entry counts, bbox_targets, means
and stds."""
import os
import pickle
import re
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from run_ref_voc_eval import _py3, xml_text  # noqa: E402

REF = "/root/reference/lib"
OUT = os.path.join(HERE, "..", "tests", "golden", "train_roidb_ref.npz")
CLASSES = ['aeroplane', 'bicycle', 'bird', 'boat', 'bottle', 'bus', 'car', 'cat', 'chair', 'cow', 'diningtable', 'dog',
           'horse', 'motorbike', 'person', 'pottedplant', 'sheep', 'sofa', 'train', 'tvmonitor']
YEARS = ('2007', '2012')
ROW_KEYS = ('boxes', 'gt_classes', 'gt_overlaps', 'max_classes', 'max_overlaps', 'bbox_targets')


def _src(path):
    src = re.sub(r"^(\s*print .*?)\s*#.*$", r"\1", open(os.path.join(REF, path)).read(), flags=re.M)  # comments after print
    return re.sub(r"\bnp\.float\b", "float", _py3(src))


def load_reference():
    """The reference's load_data namespace (load_proposal_roidb, merge_roidb, filter_roidb) with its PascalVOC, and its
    add_bbox_regression_targets."""
    sys.path.insert(0, os.path.join(HERE, "_ref"))
    import ref_bbox
    bt = {"bbox_overlaps_cython": ref_bbox.bbox_overlaps_cython,
          "ignore_overlaps_cython": ref_bbox.ignore_overlaps_cython}
    exec(compile(_src("bbox/bbox_transform.py").replace("from bbox import", "#"), "bbox_transform.py", "exec"), bt)
    im = {"__name__": "ref_imdb", "bbox_overlaps": bt["bbox_overlaps"], "ignore_overlaps": bt["ignore_overlaps"]}
    exec(compile(_src("dataset/imdb.py"), "imdb.py", "exec"), im)
    pv = {"__name__": "ref_pascal_voc", "IMDB": im["IMDB"], "voc_eval": None, "voc_eval_sds": None}
    exec(compile(_src("dataset/pascal_voc.py"), "pascal_voc.py", "exec"), pv)
    ld = {"__name__": "ref_load_data", "PascalVOC": pv["PascalVOC"]}
    exec(compile(_src("data_utils/load_data.py").replace("from dataset import *", ""), "load_data.py", "exec"), ld)
    br = {"__name__": "ref_bbox_regression"}
    exec(compile(_src("bbox/bbox_regression.py").replace("from bbox_transform import bbox_overlaps, bbox_transform", ""),
                 "bbox_regression.py", "exec"), br)
    br.update(bbox_overlaps=bt["bbox_overlaps"], bbox_transform=bt["bbox_transform"])
    return ld, br


# --------------------------------------------------------------------------------------------------------------------
# the devkit: per year, images with a few objects (some difficult), one without objects and one with only difficult
# ones (both dropped by filter_roidb when only_gt; with proposals only the one without overlapping proposals is)
# --------------------------------------------------------------------------------------------------------------------
def make_devkit(rng):
    sets = {}
    for y, year in enumerate(YEARS):
        names = ['%s_%06d' % (year, 11 * k + 5 + y) for k in range(6 + 2 * y)]
        imgs = []
        for k, name in enumerate(names):
            W, H = int(rng.randint(160, 500)), int(rng.randint(120, 400))
            objs = []
            n = 0 if k == 1 else int(rng.randint(1, 6))
            for j in range(n):
                w, h = rng.randint(8, W // 2), rng.randint(8, H // 2)
                x, y0 = rng.randint(1, W - w), rng.randint(1, H - h)
                diff = 1 if k == 2 else int(rng.rand() < 0.2)
                objs.append((CLASSES[rng.randint(20)], diff, str(x), str(y0), str(x + w), str(y0 + h)))
            imgs.append((name, W, H, objs))
        sets[year] = imgs
    return sets


def make_proposals(rng, imgs):
    """NMS-ed proposals ([n, 5] float32, score last) of every image: random boxes, one equal to the image's first
    non-difficult GT box (0-based, as load_pascal_annotation makes it), some overlapping the GT; an image without any."""
    out = []
    for k, (name, W, H, objs) in enumerate(imgs):
        n = 0 if k == 3 else int(rng.randint(3, 25))
        b = np.zeros((n, 5), np.float32)
        if n:
            x1, y1 = rng.uniform(0, W - 10, n), rng.uniform(0, H - 10, n)
            b[:, 0], b[:, 1] = x1, y1
            b[:, 2], b[:, 3] = np.minimum(x1 + rng.uniform(4, W / 2, n), W - 1), np.minimum(y1 + rng.uniform(4, H / 2, n), H - 1)
            gts = [o for o in objs if o[1] == 0]
            for j, o in enumerate(gts[:n // 2]):
                g = np.array([float(v) - 1 for v in o[2:]], np.float32)
                b[j, :4] = g if j == 0 else np.clip(g + rng.uniform(-6, 6, 4).astype(np.float32), 0, [W - 1, H - 1] * 2)
            b[:, 4] = rng.uniform(0, 1, n).astype(np.float32)
        out.append(b)
    return out


def write_devkit(root, sets, props):
    """VOCdevkit/VOC<year>/{Annotations, ImageSets/Main/trainval.txt, JPEGImages} (empty image files) and the
    proposal caches under root/proposals; returns (devkit path, proposal path)."""
    dk = os.path.join(root, 'VOCdevkit')
    pp = os.path.join(root, 'proposals')
    os.makedirs(pp, exist_ok=True)
    for year, imgs in sets.items():
        vp = os.path.join(dk, 'VOC' + year)
        for sub in ('Annotations', 'ImageSets/Main', 'JPEGImages'):
            os.makedirs(os.path.join(vp, sub), exist_ok=True)
        with open(os.path.join(vp, 'ImageSets', 'Main', 'trainval.txt'), 'w') as f:
            f.write(''.join(n + '\n' for n, _, _, _ in imgs))
        for name, W, H, objs in imgs:
            with open(os.path.join(vp, 'Annotations', name + '.xml'), 'w') as f:
                f.write(xml_text(objs, W, H))
            open(os.path.join(vp, 'JPEGImages', name + '.jpg'), 'w').close()
        with open(os.path.join(pp, 'PASCALVOC_%s_trainval_rpn_after_nms.pkl' % year), 'wb') as f:
            pickle.dump([props[year], []], f, 2)
    return dk, pp


def config(precomputed, agnostic):
    S = types.SimpleNamespace
    return S(CLASS_AGNOSTIC=agnostic,
             TRAIN=S(FG_THRESH=0.5, BG_THRESH_HI=0.5, BG_THRESH_LO=0.0, BBOX_REGRESSION_THRESH=0.5,
                     BBOX_NORMALIZATION_PRECOMPUTED=precomputed, BBOX_MEANS=[0.0, 0.0, 0.0, 0.0],
                     BBOX_STDS=[0.1, 0.1, 0.2, 0.2]))


CASES = [(mode, pre, agn) for mode in ('gt', 'rpn') for pre in (True, False) for agn in (True, False)]


def case_name(mode, pre, agn):
    return '%s_%s_%s' % (mode, 'pre' if pre else 'acc', 'agnostic' if agn else 'perclass')


def record(out, k, roidb, means, stds, dk):
    out[k + '_n'] = np.array([len(r['boxes']) for r in roidb], np.int64)
    out[k + '_image'] = np.array([os.path.relpath(r['image'], dk) for r in roidb])
    out[k + '_flipped'] = np.array([r['flipped'] for r in roidb])
    out[k + '_hw'] = np.array([[r['height'], r['width']] for r in roidb], np.float64)
    for key in ROW_KEYS:
        out[k + '_' + key] = np.concatenate([np.asarray(r[key]) for r in roidb])
    out[k + '_means'], out[k + '_stds'] = np.asarray(means), np.asarray(stds)


def main():
    ld, br = load_reference()
    rng = np.random.RandomState(0)
    sets = make_devkit(rng)
    props = {year: make_proposals(rng, imgs) for year, imgs in sets.items()}
    out = {}
    for year, imgs in sets.items():
        out['devkit_%s_names' % year] = np.array([n for n, _, _, _ in imgs])
        out['devkit_%s_xml' % year] = np.array([xml_text(o, W, H) for _, W, H, o in imgs])
        for i, p in enumerate(props[year]):
            out['props_%s_%d' % (year, i)] = p
    for mode, pre, agn in CASES:
        with tempfile.TemporaryDirectory() as root:
            dk, pp = write_devkit(root, sets, props)
            roidbs = [ld['load_proposal_roidb']('PascalVOC', year + '_trainval', root, dk, proposal='rpn',
                                                append_gt=True, flip=True, proposal_path=pp, only_gt=mode == 'gt')
                      for year in YEARS]
            roidb = ld['filter_roidb'](ld['merge_roidb'](roidbs), config(pre, agn))
            means, stds = br['add_bbox_regression_targets'](roidb, config(pre, agn))
            record(out, case_name(mode, pre, agn), roidb, means, stds, dk)
        print(case_name(mode, pre, agn), 'entries', len(roidb), 'rows', int(out[case_name(mode, pre, agn) + '_n'].sum()))
    np.savez_compressed(OUT, **out)
    print('wrote', os.path.relpath(OUT), os.path.getsize(OUT), 'bytes')


if __name__ == "__main__":
    sys.exit(main())
