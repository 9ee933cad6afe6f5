"""Negative-chip proposal pipeline on the device: the batched proposal NMS (sniper_proposal_nms_batched) against the
reference's own nmsp (tests/golden/proposals_ref.npz) and the numpy restatement with its tie rule; proposal extraction
(MNIteratorTest + Tester.extract_proposals on forward_rpn) against forward_rpn on each image alone; and the loaded
proposal roidb driving negative-chip training steps."""
import math
import os
import pickle
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
GOLD = os.path.join(ROOT, "tests", "golden", "proposals_ref.npz")


def _device_keeps(cases):
    import torch
    from sniper_b200 import proposals as PR
    keeps = PR.nms_keeps([np.ascontiguousarray(c, dtype=np.float32) for c in cases], device="cuda")
    torch.cuda.synchronize()
    return keeps


def test_proposal_nms_matches_reference_nmsp():
    """Every fixture image in one launch: tie-free random images, IoU exactly float32(0.7) and just above, 0 / 1 / 4096
    rows; keep lists bit-identical to the reference's nmsp."""
    g = np.load(GOLD)
    cases = [g["nms_dets_%d" % c] for c in range(int(g["nms_n"]))]
    for c, k in enumerate(_device_keeps(cases)):
        assert np.array_equal(k, g["nms_keep_%d" % c]), c


def test_proposal_nms_ties_match_restatement():
    """Tie-heavy and MultiProposal-filler-like inputs (repeated boxes at score 0) against the numpy restatement's rule:
    exact score ties go to the higher row.  Also several chunks of images."""
    import proposal_nms_np as PN
    from sniper_b200 import proposals as PR
    rng = np.random.RandomState(3)
    cases = []
    for n in (3, 17, 300, 900, 2000):
        xy = rng.randint(0, 60, (n, 2)).astype(np.float32) * 8
        wh = rng.randint(1, 6, (n, 2)).astype(np.float32) * 16
        d = np.concatenate([xy, xy + wh, (rng.randint(0, 4, (n, 1)) / 4.0).astype(np.float32)], 1)
        cases.append(d)
    for n_real, n_fill in ((0, 5), (120, 180), (290, 10)):
        real = cases[2][:n_real].copy()
        fill = np.tile(np.array([[0, 0, 15, 15, 0]], np.float32), (n_fill, 1))
        cases.append(np.concatenate([real, fill], 0))
    keeps = PR.nms_keeps(cases, device="cuda", chunk=3)
    for c, (d, k) in enumerate(zip(cases, keeps)):
        assert np.array_equal(k, PN.nmsp_keep(d)), c
    assert any(len(k) < len(d) for d, k in zip(cases, keeps))


def test_proposal_nms_refuses_oversized_and_negative_inputs():
    import torch
    from sniper_b200 import ops
    from sniper_b200._lib import SniperError
    rng = np.random.RandomState(1)
    ok = rng.uniform(0, 100, (10, 5)).astype(np.float32)
    big = rng.uniform(0, 100, (4097, 5)).astype(np.float32)
    with pytest.raises(SniperError, match="image 1 has 4097 rows"):
        ops.proposal_nms_batched(torch.from_numpy(np.concatenate([ok, big])).cuda(), [0, 10, 10 + 4097])
    neg = ok.copy()
    neg[4, 4] = -0.5
    with pytest.raises(SniperError, match="image 2 has a negative score"):
        ops.proposal_nms_batched(torch.from_numpy(np.concatenate([ok, ok, neg])).cuda(), [0, 10, 20, 30])


# ---------------------------------------------------------------- extraction and training on the loaded proposals
SCALES = [(96, 160), (128, 224)]


def _config():
    from sniper_b200 import iterator as IT
    cfg = IT.default_config(neg=True)
    cfg.TEST.SCALES = SCALES
    cfg.TEST.BATCH_IMAGES = [2, 3]
    cfg.dataset.dataset, cfg.dataset.test_image_set = "synthetic", "train"
    return cfg


def _gt_roidb():
    from sniper_b200 import iterator as IT
    gt = IT.synthetic_roidb(5, seed=11, n_prop=0, n_gt=(2, 8))
    for r in gt:
        r['flipped'] = False
        r['gt_classes'] = r['max_classes'].astype(np.int32)
        r['gt_overlaps'] = np.zeros((len(r['boxes']), 81), np.float32)
        r['gt_overlaps'][np.arange(len(r['boxes'])), r['gt_classes']] = 1
    return gt


@pytest.fixture(scope="module")
def trainer():
    from sniper_b200 import model, synth_batch, trainer as TR
    mc = model.Cfg()
    mc.batch_images = 2
    tr = TR.Trainer(mc, device="cuda:0", scheduler=None, seed=3, deform_offset_std=0.01)
    tr.net.train_step(synth_batch.make_batch(2, seed=7, device="cuda"), lr=0.001)      # non-trivial moving statistics
    return tr


def test_extracted_proposals_equal_forward_rpn_per_image(trainer, tmp_path):
    """imdb_proposal_extraction_wrapper over both scales: each image's proposals at each scale equal forward_rpn on that
    image alone (its own batch of one, same canvas), / float32 scale, first 300 rows, bit for bit; the pickle reads
    back.  The rows after an image's proposals are MultiProposal's score-0 filler, whose boxes depend on the image's
    position in its batch: only their number and zero scores are compared."""
    import torch
    from sniper_b200 import tester as TS
    net, cfg, db = trainer.net, _config(), _gt_roidb()
    final, stats = TS.imdb_proposal_extraction_wrapper(net, cfg, db, str(tmp_path))
    assert [s['scale'] for s in stats['scales']] == SCALES
    with open(os.path.join(str(tmp_path), "SYNTHETIC_train_rpn.pkl"), "rb") as f:
        back = pickle.load(f, encoding="latin1")
    assert len(back) == len(db) and all(a.tobytes() == b.tobytes() for a, b in zip(back, final))
    n_real = 0
    for i, r in enumerate(db):
        assert final[i].dtype == np.float32 and final[i].shape == (600, 5)
        for k, scale in enumerate(SCALES):
            b = next(TS.MNIteratorTest([r], cfg, scale, batch_size=1))
            rois, sc = net.forward_rpn(b['data'], b['im_info'])
            s = np.float32(b['im_info'][0, 2].item())
            rois, sc = rois.cpu().numpy(), sc.cpu().numpy()
            want = np.hstack((rois[:300, 1:] / s, sc[:300, None])).astype(np.float32)
            got = final[i][300 * k:300 * (k + 1)]
            kept = int(np.argmin(np.append(want[:, 4] > 0, False)))        # the filler follows the proposals
            assert (want[kept:, 4] == 0).all() and (got[kept:, 4] == 0).all() and (got[:kept, 4] > 0).all(), (i, k)
            assert got[:kept].tobytes() == want[:kept].tobytes(), (i, k)
            n_real += kept
    torch.cuda.synchronize()
    assert n_real > 0


def test_rpn_roidb_trains_on_negative_chips(trainer, tmp_path):
    """Extracted proposals -> rpn_roidb (device NMS, cache) -> MNIteratorE2E(USE_NEG_CHIPS) -> two Trainer.step_raw."""
    import proposal_nms_np as PN
    from sniper_b200 import iterator as IT
    from sniper_b200 import proposals as PR
    from sniper_b200 import tester as TS
    cfg, gt = _config(), _gt_roidb()
    raw_props, _ = TS.imdb_proposal_extraction_wrapper(trainer.net, cfg, gt, str(tmp_path))
    imdb = PR.IMDB("SYNTHETIC_train", 81)
    roidb = imdb.rpn_roidb(gt, append_gt=True, proposal_path=str(tmp_path))
    assert os.path.exists(os.path.join(str(tmp_path), "SYNTHETIC_train_rpn_after_nms.pkl"))
    cached, _ = imdb.load_rpn_data(str(tmp_path))
    for p, c in zip(raw_props, cached):
        assert c.tobytes() == p[PN.nmsp_keep(p)].tobytes()
    for r in roidb:
        assert len(r['boxes']) == len(r['gt_classes']) == len(r['max_overlaps']) == len(r['proposal_scores'])
    np.random.seed(2)
    it = IT.MNIteratorE2E(roidb, cfg, batch_size=2)
    assert sum(len(r['neg_crops']) for r in roidb) > 0
    stage = IT.InputStage(cfg, "cuda:0", 2)
    for _ in range(2):
        out = trainer.step_raw(next(it), stage, lr=0.001)
        assert all(math.isfinite(v) for v in out.values()), out
