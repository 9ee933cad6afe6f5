"""The training roidb from an image set on disk, in main_train.py's order (:49-70):

    paper_train_scales(config)
    roidbs = [load_proposal_roidb(dataset, image_set, root_path, dataset_path, flip=config.TRAIN.FLIP,
                                  proposal_path=..., only_gt=not config.TRAIN.USE_NEG_CHIPS)
              for image_set in image_sets.split('+')]
    roidb = filter_roidb(merge_roidb(roidbs), config)
    bbox_means, bbox_stds = add_bbox_regression_targets(roidb, config)

Mirror of lib/data_utils/load_data.py, `append_flipped_images` of lib/dataset/imdb.py (:214-272, without the mask
branch) and lib/bbox/bbox_regression.py (:18-116): same names, field names, dtypes and entry order (the reference's own
code on seeded inputs is tests/golden/train_roidb_ref.npz).  `dataset` is the name the configs use: 'coco'
(`coco.coco`) or 'PascalVOC' (`pascal_voc.PascalVOC`).  The proposal NMS of the rpn_roidb branch runs on the device
(`proposals.IMDB`); the rest is one-time host preparation, as in the reference.

One addition: an entry that carries decoded pixels ('image_data') shares the array with its flipped copy; the iterator
mirrors the pixels of `flipped` entries on the device (`sniper_chip_input`), as it does for entries read from a path.
"""
import time

import numpy as np

from . import coco, host, pascal_voc, proposals

DATASETS = {'coco': coco.coco, 'PascalVOC': pascal_voc.PascalVOC}
PAPER_COCO_SCALES = (3.0, 1.667, 512.0)


def paper_train_scales(config):
    """main_train.py:46-52: a COCO config with 81 classes trains at the paper's scales (3.0, 1.667, 512.0) -- factors,
    the last one the longer side in pixels (chip_worker.image_scales) -- whatever its TRAIN.SCALES say.  Sets
    config.TRAIN.SCALES and returns it."""
    if config.dataset.dataset == 'coco' and config.dataset.NUM_CLASSES == 81:
        config.TRAIN.SCALES = PAPER_COCO_SCALES
    return config.TRAIN.SCALES


def _imdb(dataset_name, image_set_name, root_path, dataset_path, result_path, device):
    if dataset_name not in DATASETS:
        raise ValueError("dataset must be one of %s, not %r" % (sorted(DATASETS), dataset_name))
    return DATASETS[dataset_name](image_set_name, root_path, dataset_path, result_path, device=device)


def append_flipped_images(imdb, roidb):
    """Appends a horizontally flipped copy of every entry (imdb.py:214-272): boxes x -> width - x - 1, the class and
    overlap arrays and proposal_scores shared with the source entry, 'flipped': True.  The pixels are flipped when the
    chips are loaded.  imdb.num_images becomes the entry count before the flip and imdb.image_set_index is doubled, as
    in the reference."""
    entries = len(roidb)
    imdb.num_images = entries
    for i in range(entries):
        roi_rec = roidb[i]
        boxes = roi_rec['boxes'].copy()
        oldx1 = boxes[:, 0].copy()
        oldx2 = boxes[:, 2].copy()
        boxes[:, 0] = roi_rec['width'] - oldx2 - 1
        boxes[:, 2] = roi_rec['width'] - oldx1 - 1
        if not (boxes[:, 2] >= boxes[:, 0]).all():
            raise ValueError("append_flipped_images: entry %d (%s) has a box outside its width %s"
                             % (i, roi_rec.get('image'), roi_rec['width']))
        entry = {'image': roi_rec['image'],
                 'height': roi_rec['height'],
                 'width': roi_rec['width'],
                 'boxes': boxes,
                 'gt_classes': roi_rec['gt_classes'],
                 'gt_overlaps': roi_rec['gt_overlaps'],
                 'max_classes': roi_rec['max_classes'],
                 'max_overlaps': roi_rec['max_overlaps'],
                 'flipped': True}
        if 'proposal_scores' in roi_rec:
            entry['proposal_scores'] = roi_rec['proposal_scores']
        if 'image_data' in roi_rec:
            entry['image_data'] = roi_rec['image_data']
        roidb.append(entry)
    imdb.image_set_index *= 2
    return roidb


def load_gt_roidb(dataset_name, image_set_name, root_path, dataset_path, result_path=None, flip=False, device="cuda"):
    """The GT roidb of one image set (load_data.py:13-20), flipped copies appended when flip."""
    imdb = _imdb(dataset_name, image_set_name, root_path, dataset_path, result_path, device)
    roidb = imdb.gt_roidb()
    if flip:
        roidb = append_flipped_images(imdb, roidb)
    return roidb


def load_proposal_roidb(dataset_name, image_set_name, root_path, dataset_path, result_path=None, proposal='rpn',
                        append_gt=True, flip=False, proposal_path='proposals', only_gt=False, get_imdb=False,
                        device="cuda", times=None):
    """The training roidb of one image set (load_data.py:23-42).  only_gt: the GT roidb with float32 boxes; otherwise
    the RPN proposals of `<imdb.name>_rpn.pkl` under proposal_path, NMS-ed on the device and appended to the GT rows
    (proposals.IMDB.rpn_roidb).  flip: flipped copies appended.  get_imdb: returns (roidb, imdb).  times, when a dict,
    gets the seconds spent reading the GT (gt_s), building the proposal rows (rpn_s: the proposal file, its NMS and the
    overlaps with the GT) and flipping (flip_s)."""
    if proposal != 'rpn':
        raise ValueError("load_proposal_roidb: proposal must be 'rpn', not %r" % (proposal,))
    t0 = time.time()
    imdb = _imdb(dataset_name, image_set_name, root_path, dataset_path, result_path, device)
    roidb = imdb.gt_roidb()
    t1 = time.time()
    if not only_gt:
        roidb = proposals.IMDB(imdb.name, imdb.num_classes, device=device).rpn_roidb(roidb, append_gt,
                                                                                     proposal_path=proposal_path)
    else:
        for r in roidb:
            r['boxes'] = r['boxes'].astype(np.float32)
    t2 = time.time()
    if flip:
        roidb = append_flipped_images(imdb, roidb)
    if times is not None:
        times.update(gt_s=t1 - t0, rpn_s=t2 - t1, flip_s=time.time() - t2)
    return (roidb, imdb) if get_imdb else roidb


def merge_roidb(roidbs):
    """The roidbs one after the other, in the first list (load_data.py:45-50)."""
    roidb = roidbs[0]
    for r in roidbs[1:]:
        roidb.extend(r)
    return roidb


def filter_roidb(roidb, config):
    """The entries with at least one foreground (max_overlaps >= TRAIN.FG_THRESH) or background row (in
    [TRAIN.BG_THRESH_LO + 0.0001, TRAIN.BG_THRESH_HI)), in order (load_data.py:87-108)."""
    tr = config.TRAIN

    def is_valid(entry):
        overlaps = entry['max_overlaps']
        fg_inds = np.where(overlaps >= tr.FG_THRESH)[0]
        bg_inds = np.where((overlaps < tr.BG_THRESH_HI) & (overlaps >= tr.BG_THRESH_LO + 0.0001))[0]
        return len(fg_inds) > 0 or len(bg_inds) > 0

    num = len(roidb)
    filtered_roidb = [entry for entry in roidb if is_valid(entry)]
    print('filtered %d roidb entries: %d -> %d' % (num - len(filtered_roidb), num, len(filtered_roidb)))
    return filtered_roidb


def bbox_transform(ex_rois, gt_rois):
    """The (dx, dy, dw, dh) regression targets from ex_rois to gt_rois, float64 [N, 4] (bbox_transform.py:64-90): centre
    offsets over the source size and log size ratios, sizes with the +1 pixel convention and 1e-7 under divisions."""
    ex_w = ex_rois[:, 2] - ex_rois[:, 0] + 1.0
    ex_h = ex_rois[:, 3] - ex_rois[:, 1] + 1.0
    ex_cx = ex_rois[:, 0] + 0.5 * (ex_w - 1.0)
    ex_cy = ex_rois[:, 1] + 0.5 * (ex_h - 1.0)
    gt_w = gt_rois[:, 2] - gt_rois[:, 0] + 1.0
    gt_h = gt_rois[:, 3] - gt_rois[:, 1] + 1.0
    gt_cx = gt_rois[:, 0] + 0.5 * (gt_w - 1.0)
    gt_cy = gt_rois[:, 1] + 0.5 * (gt_h - 1.0)
    return np.stack([(gt_cx - ex_cx) / (ex_w + 1e-7), (gt_cy - ex_cy) / (ex_h + 1e-7), np.log(gt_w / (ex_w + 1e-7)),
                     np.log(gt_h / (ex_h + 1e-7))], axis=1)


def compute_bbox_regression_targets(rois, overlaps, labels, cfg):
    """[k, 5] float32 (class, dx, dy, dw, dh) of one entry (bbox_regression.py:18-52): every row with overlap >=
    TRAIN.BBOX_REGRESSION_THRESH regresses to the GT row (overlap == 1) it overlaps most, the first one on ties."""
    rois = rois.astype(np.float64, copy=False)
    if len(rois) != len(overlaps):
        raise ValueError("bbox regression: %d rois and %d overlaps" % (len(rois), len(overlaps)))
    gt_inds = np.where(overlaps == 1)[0]
    ex_inds = np.where(overlaps >= cfg.TRAIN.BBOX_REGRESSION_THRESH)[0]
    targets = np.zeros((rois.shape[0], 5), dtype=np.float32)
    if len(ex_inds) == 0:
        return targets
    ex_gt_overlaps = host.bbox_overlaps(rois[ex_inds, :], rois[gt_inds, :])
    gt_assignment = ex_gt_overlaps.argmax(axis=1)
    targets[ex_inds, 0] = labels[ex_inds]
    targets[ex_inds, 1:] = bbox_transform(rois[ex_inds, :], rois[gt_inds[gt_assignment], :])
    return targets


def add_bbox_regression_targets(roidb, cfg):
    """Adds 'bbox_targets' to every entry and normalises them per class (bbox_regression.py:55-116): by
    TRAIN.BBOX_MEANS / BBOX_STDS when TRAIN.BBOX_NORMALIZATION_PRECOMPUTED, else by the mean and standard deviation
    of the targets of each class over the roidb.  CLASS_AGNOSTIC: one foreground class.  Returns (means.ravel(),
    stds.ravel()), [num_classes * 4] float64 each."""
    if len(roidb) == 0 or 'max_classes' not in roidb[0]:
        raise ValueError("add_bbox_regression_targets: an empty roidb or one without max_classes")
    num_classes = 2 if cfg.CLASS_AGNOSTIC else roidb[0]['gt_overlaps'].shape[1]
    for r in roidb:
        r['bbox_targets'] = compute_bbox_regression_targets(r['boxes'], r['max_overlaps'], r['max_classes'], cfg)

    def rows(targets, cls):
        return np.where(targets[:, 0] > 0)[0] if cfg.CLASS_AGNOSTIC else np.where(targets[:, 0] == cls)[0]

    if cfg.TRAIN.BBOX_NORMALIZATION_PRECOMPUTED:
        means = np.tile(np.array(cfg.TRAIN.BBOX_MEANS), (num_classes, 1))
        stds = np.tile(np.array(cfg.TRAIN.BBOX_STDS), (num_classes, 1))
    else:
        class_counts = np.zeros((num_classes, 1)) + 1e-14
        sums = np.zeros((num_classes, 4))
        squared_sums = np.zeros((num_classes, 4))
        for r in roidb:
            targets = r['bbox_targets']
            for cls in range(1, num_classes):
                cls_indexes = rows(targets, cls)
                if cls_indexes.size > 0:
                    class_counts[cls] += cls_indexes.size
                    sums[cls, :] += targets[cls_indexes, 1:].sum(axis=0)
                    squared_sums[cls, :] += (targets[cls_indexes, 1:] ** 2).sum(axis=0)
        means = sums / class_counts
        # var(x) = E(x^2) - E(x)^2
        stds = np.sqrt(squared_sums / class_counts - means ** 2)
    for r in roidb:
        targets = r['bbox_targets']
        for cls in range(1, num_classes):
            cls_indexes = rows(targets, cls)
            targets[cls_indexes, 1:] -= means[cls, :]
            targets[cls_indexes, 1:] /= stds[cls, :]
    return means.ravel(), stds.ravel()
