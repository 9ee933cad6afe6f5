"""Host half of the negative-chip proposal pipeline against the reference's own code (tests/golden/proposals_ref.npz,
written by oracle/run_ref_proposals.py): the numpy restatement of nmsp, the proposal roidb and its merge into the GT
roidb (sniper_b200/proposals.py), the proposal arithmetic of Tester.extract_proposals and the batch order of
MNIteratorTest (sniper_b200/tester.py); then the proposal cache round trip and one MNIteratorE2E epoch with negative
chips on a merged roidb."""
import copy
import os
import pickle
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import proposal_nms_np as PN  # noqa: E402
from sniper_b200 import iterator as IT  # noqa: E402
from sniper_b200 import proposals as PR  # noqa: E402
from sniper_b200 import tester as TS  # noqa: E402

GOLD = np.load(os.path.join(ROOT, "tests", "golden", "proposals_ref.npz"))
NUM_CLASSES = 21


def _gt_roidb(n):
    out = []
    for i in range(n):
        boxes, cls = GOLD["roidb_gt_boxes_%d" % i], GOLD["roidb_gt_classes_%d" % i]
        ov = np.zeros((len(cls), NUM_CLASSES), np.float32)
        ov[np.arange(len(cls)), cls] = 1
        out.append(dict(image="im%d.jpg" % i, width=1333, height=800, boxes=boxes, gt_classes=cls, gt_overlaps=ov,
                        max_classes=cls.copy(), max_overlaps=np.ones(len(cls), np.float32), flipped=False))
    return out


def test_nmsp_restatement_matches_reference():
    """Tie-free random images, pairs at IoU exactly float32(0.7) and just above, 0 / 1 / 4096 rows."""
    for c in range(int(GOLD["nms_n"])):
        keep = PN.nmsp_keep(GOLD["nms_dets_%d" % c])
        assert np.array_equal(keep, GOLD["nms_keep_%d" % c]), c


def test_nmsp_restatement_breaks_ties_to_the_higher_row():
    d = np.array([[0, 0, 9, 9, 0.5], [0, 0, 9, 9, 0.5], [100, 100, 120, 120, 0.5], [0, 0, 9, 9, 0.9]], np.float32)
    assert PN.nmsp_keep(d).tolist() == [3, 2]


def test_proposal_roidb_and_merge_match_reference():
    """create_roidb_from_box_list + merge_roidbs field by field, bit for bit; proposal_scores is the one deliberate
    difference: the reference keeps only the GT rows' 10s, here each proposal row's score follows them."""
    n = int(GOLD["roidb_n"])
    props = [GOLD["roidb_props_%d" % i] for i in range(n)]
    gt = _gt_roidb(n)
    imdb = PR.IMDB("test", NUM_CLASSES)
    rpn = imdb.create_roidb_from_box_list(props, [], gt)
    merged = PR.IMDB.merge_roidbs(copy.deepcopy(gt), rpn)
    for i, m in enumerate(merged):
        for k in ("boxes", "gt_classes", "gt_overlaps", "max_classes", "max_overlaps"):
            ref = GOLD["roidb_merged_%s_%d" % (k, i)]
            assert m[k].dtype == ref.dtype and m[k].shape == ref.shape and m[k].tobytes() == ref.tobytes(), (i, k)
        ng = len(gt[i]['boxes'])
        assert GOLD["roidb_merged_proposal_scores_%d" % i].tolist() == [10.0] * ng
        want = np.hstack((10 * np.ones(ng), GOLD["roidb_rpn_scores_%d" % i]))
        assert m['proposal_scores'].shape == (len(m['boxes']),) and np.array_equal(m['proposal_scores'], want)
    # a proposal equal to a GT box is labelled like a GT row (max_overlaps == 1), as in the reference
    assert any((m['max_overlaps'][len(g['boxes']):] == 1).any() for m, g in zip(merged, gt))
    # images without GT: background proposals only
    assert all((m['max_classes'] == 0).all() for m, g in zip(merged, gt) if len(g['boxes']) == 0)


def test_extract_proposals_host_arithmetic_matches_reference():
    """Tester.get_proposals / extract_proposals on fixed RPN outputs: rois / float32 scale, first n rows, score last."""
    rois, scores = GOLD["ext_rois"], GOLD["ext_scores"]
    im_info, im_ids = GOLD["ext_im_info"], GOLD["ext_im_ids"]

    class Net(object):
        def forward_rpn(self, data, info):
            return torch.from_numpy(rois), torch.from_numpy(scores)
    batch = dict(data=torch.zeros(len(im_ids), 3, 1, 1), im_info=torch.from_numpy(im_info), im_ids=im_ids)
    tester = TS.Tester(Net(), None, [None] * 3, [batch], None, batch_size=3, num_classes=1)
    boxes = tester.extract_proposals(n_proposals=25)
    for i in range(3):
        ref = GOLD["ext_boxes_%d" % i]
        assert boxes[i].dtype == np.float32 and boxes[i].shape == ref.shape == (25, 5)
        assert boxes[i].tobytes() == ref.tobytes(), i


def test_mniterator_test_order_and_fixed_canvas():
    """MNIteratorTest.reset's order (horizontal, then vertical, each padded with its first image); every batch of an
    orientation has the same canvas."""
    cfg = IT.default_config()
    for c in range(int(GOLD["iter_n"])):
        wh, bs = GOLD["iter_wh_%d" % c], int(GOLD["iter_bs_%d" % c])
        db = [dict(width=int(w), height=int(h)) for w, h in wh]
        it = TS.MNIteratorTest(db, cfg, (800, 1280), batch_size=bs, device="cpu")
        assert it.inds.tolist() == GOLD["iter_inds_%d" % c].tolist(), c
    rng = np.random.RandomState(0)
    db = [dict(width=w, height=h, image_data=rng.randint(0, 256, (h, w, 3)).astype(np.uint8))
          for w, h in ((300, 200), (320, 160), (200, 300), (150, 310), (240, 240))]
    it = TS.MNIteratorTest(db, cfg, (96, 160), batch_size=2, device="cpu")
    canv = [(b['canvas'], [db[i]['width'] >= db[i]['height'] for i in b['im_ids']]) for b in it]
    assert [c for c, _ in canv] == [(96, 256), (96, 256), (160, 128)]
    assert [h for _, h in canv] == [[True, True], [True, True], [False, False]]
    for b in TS.MNIteratorTest(db, cfg, (96, 160), batch_size=2, device="cpu"):
        for k, i in enumerate(b['im_ids']):
            s = TS.chips_inference.image_scale(db[i]['width'], db[i]['height'], (96, 160))
            assert b['im_info'][k, 2].item() == np.float32(s)
            assert b['im_info'][k, 0].item() == np.rint(db[i]['height'] * s)


def test_proposal_cache_round_trip(tmp_path):
    """load_rpn_data reads the `_rpn_after_nms.pkl` cache (protocol 2, as Python 2 writes it) without running the NMS."""
    boxes = [GOLD["roidb_props_%d" % i] for i in range(int(GOLD["roidb_n"]))]
    with open(os.path.join(str(tmp_path), "coco_x_rpn_after_nms.pkl"), "wb") as f:
        pickle.dump([boxes, []], f, protocol=2)
    got, maps = PR.IMDB("coco_x", NUM_CLASSES, device="cpu").load_rpn_data(str(tmp_path))
    assert maps == [] and len(got) == len(boxes)
    assert all(a.dtype == b.dtype and a.tobytes() == b.tobytes() for a, b in zip(got, boxes))


def test_merged_roidb_feeds_negative_chips():
    """One MNIteratorE2E epoch (USE_NEG_CHIPS) over GT + proposal rows: negative chips are mined from the proposals."""
    cfg = IT.default_config(neg=True)
    rng = np.random.RandomState(5)
    gt = IT.synthetic_roidb(6, seed=3, n_prop=0)
    props = []
    for r in gt:
        r['flipped'] = False
        r['gt_classes'] = r['max_classes'].astype(np.int32)
        r['gt_overlaps'] = np.zeros((len(r['boxes']), 81), np.float32)
        r['gt_overlaps'][np.arange(len(r['boxes'])), r['gt_classes']] = 1
        n = 300
        x1, y1 = rng.uniform(0, r['width'] - 40, n), rng.uniform(0, r['height'] - 40, n)
        w, h = rng.uniform(16, 200, n), rng.uniform(16, 200, n)
        p = np.stack([x1, y1, np.minimum(x1 + w, r['width'] - 1), np.minimum(y1 + h, r['height'] - 1),
                      rng.uniform(0, 1, n)], 1).astype(np.float32)
        props.append(p)
    imdb = PR.IMDB("synthetic", 81)
    roidb = PR.IMDB.merge_roidbs(gt, imdb.create_roidb_from_box_list(props, [], gt))
    np.random.seed(1)
    it = IT.MNIteratorE2E(roidb, cfg, batch_size=4)
    assert sum(len(r['neg_crops']) for r in roidb) > 0
    n_neg = sum(min(len(r['neg_crops']), 2) for r in roidb)
    assert it.chip_count == sum(len(r['crops']) for r in roidb) and n_neg > 0
    seen = sum(4 for _ in it)
    assert seen == it.size >= it.chip_count
