"""Proposal recall on the device (csrc/proposal_recall.cu) byte-equal to the reference's own IMDB.evaluate_recall
(tests/golden/recall_ref.npz) and to the numpy restatement (oracle/recall_np.py) at COCO-train proposal counts, the
worst-case image on the workspace path, and the recall of imdb_proposal_extraction_wrapper."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", "oracle"))

import recall_fixture as F  # noqa: E402
import recall_np  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return F.load()


def _device(roidb, cand, thr, n_img, **kw):
    from sniper_b200 import ops, recall
    t = recall.default_thresholds() if thr is None else thr
    return ops.proposal_recall(*recall.recall_inputs(roidb, cand, n_img), t, **kw)


def _same(res, rec, ov):
    assert res['recalls'].tobytes() == np.asarray(rec, np.float64).tobytes()
    for r in range(7):
        assert res['gt_overlaps'][r].tobytes() == ov[r].tobytes(), r


@pytest.mark.parametrize("name", F.CASES)
def test_device_equals_reference(fx, name, capsys):
    from sniper_b200 import recall
    roidb, cand, thr, n_img = F.case(fx, name)
    text, rec, ov = F.expected(fx, name)
    _same(_device(roidb, cand, thr, n_img), rec, ov)
    assert recall.evaluate_recall(roidb, cand, thr, num_images=n_img) == text
    assert capsys.readouterr().out == str(fx[name + '_stdout'])


def test_imdb_classes_delegate(fx):
    from sniper_b200 import proposals
    roidb, cand, thr, n_img = F.case(fx, "seeded")
    text = F.expected(fx, "seeded")[0]
    assert proposals.IMDB('x', 5).evaluate_recall(roidb, cand, thr) == text

    class Fake(object):
        num_images, device = n_img, "cuda"
    from sniper_b200 import coco, pascal_voc
    for cls in (coco.coco, pascal_voc.PascalVOC):
        assert cls.evaluate_recall(Fake(), roidb, cand, thr) == text


def test_device_equals_restatement_at_coco_counts():
    from sniper_b200 import recall
    roidb, cand = F.coco_like(5, 5000)
    text, want = recall_np.evaluate(roidb, cand)
    res = _device(roidb, cand, None, None)
    _same(res, want['recalls'], want['gt_overlaps'])
    assert res['ar'].tobytes() == want['ar'].tobytes()
    assert list(res['num_pos']) == list(want['num_pos']) and list(res['area_counts']) == list(want['area_counts'])
    assert recall.evaluate_recall(roidb, cand, verbose=False) == text


def test_worst_case_image_runs_on_the_workspace():
    from sniper_b200 import _lib, recall
    rng = np.random.RandomState(3)
    roidb, cand = F.coco_like(9, 3, props=(6000, 6001), big=(100, 101), crowded=1.0)
    # duplicate GTs and proposals: ties everywhere in the rescans
    roidb[0]['boxes'][1::2] = roidb[0]['boxes'][0::2][:len(roidb[0]['boxes'][1::2])]
    cand[1][rng.randint(6000, size=3000)] = cand[1][rng.randint(6000, size=3000)]
    prop_box, prop_off, gt_box, gt_off, gt_range = recall.recall_inputs(roidb, cand)
    ws = np.zeros(7 * 3 + 1, np.int64)
    assert _lib.lib().sniper_proposal_recall_workspace_bytes(
        prop_off.astype(np.int32).ctypes.data, gt_off.astype(np.int32).ctypes.data, gt_range.ctypes.data, 3,
        ws.ctypes.data) == 0
    assert ws[1] - ws[0] == 6000 * (gt_off[1] - gt_off[0]) * 8        # image 0, range all: the workspace
    text, want = recall_np.evaluate(roidb, cand)
    for budget in (1 << 30, 1):                                       # one launch; one launch per pair
        _same(_device(roidb, cand, None, None, max_workspace_bytes=budget), want['recalls'], want['gt_overlaps'])


def test_extraction_wrapper_scores_its_proposals(tmp_path):
    import torch
    from sniper_b200 import iterator as IT
    from sniper_b200 import model, proposals, recall, synth_batch
    from sniper_b200 import tester as TS
    from sniper_b200 import trainer as TR
    cfg = IT.default_config(neg=True)
    cfg.TEST.SCALES = [(96, 160), (128, 224)]
    cfg.TEST.BATCH_IMAGES = [2, 3]
    cfg.dataset.dataset, cfg.dataset.test_image_set = "synthetic", "train"
    db = IT.synthetic_roidb(5, seed=11, n_prop=0, n_gt=(2, 8))
    for r in db:
        r['flipped'] = False
        r['gt_classes'] = r['max_classes'].astype(np.int32)
        r['gt_overlaps'] = np.zeros((len(r['boxes']), 81), np.float32)
        r['gt_overlaps'][np.arange(len(r['boxes'])), r['gt_classes']] = 1
    mc = model.Cfg()
    mc.batch_images = 2
    tr = TR.Trainer(mc, device="cuda:0", scheduler=None, seed=3, deform_offset_std=0.01)
    tr.net.train_step(synth_batch.make_batch(2, seed=7, device="cuda"), lr=0.001)
    plain, s0 = TS.imdb_proposal_extraction_wrapper(tr.net, cfg, db, str(tmp_path / "a"))
    final, s1 = TS.imdb_proposal_extraction_wrapper(tr.net, cfg, db, str(tmp_path / "b"),
                                                    imdb=proposals.IMDB('synthetic', 81))
    torch.cuda.synchronize()
    assert 'recall' not in s0 and set(s1) == set(s0) | {'recall', 'recall_s'}
    assert all(a.tobytes() == b.tobytes() for a, b in zip(plain, final))
    assert s1['recall'] == recall.evaluate_recall(db, [p[:, :4] for p in final], verbose=False)
    assert s1['recall'] == recall_np.evaluate(db, [p[:, :4] for p in final])[0]
