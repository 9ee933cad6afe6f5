"""COCO box evaluation on the device (csrc/coco_eval.cu through sniper_b200.cocoeval): bit for bit against the
reference's own pycocotools on the fixture cases (tests/golden/cocoeval_ref.npz), and against the numpy restatement
(oracle/cocoeval_np.py) on seeded sets up to val2017's shape; then the COCO imdb and the test wrapper end to end."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", "oracle"))

import cocoeval_fixture as F  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return F.load()


def _evaluated(cg, cd, p):
    from sniper_b200 import cocoeval
    E = cocoeval.COCOeval(cg, cd)
    E.params.iouThrs, E.params.recThrs, E.params.maxDets, E.params.areaRng = p.iouThrs, p.recThrs, p.maxDets, p.areaRng
    E.evaluate()
    E.accumulate()
    return E


@pytest.mark.parametrize("name", F.CASES)
def test_device_equals_reference(fx, name):
    E = _evaluated(*F.cocos(fx, name))
    assert E.eval['precision'].tobytes() == fx[name + "_precision"].tobytes()
    assert E.eval['recall'].tobytes() == fx[name + "_recall"].tobytes()
    assert E.eval['counts'] == list(fx[name + "_precision"].shape)
    if name + "_stats" in fx:
        assert np.asarray(E.summarize()).tobytes() == fx[name + "_stats"].tobytes()
    F.assert_evalimgs_equal(F.flat_evalimgs(E.evalImgs), fx, name)
    # ious: bbIou bit for bit, keyed (imgId, catId), [] for the empty pairs
    keys = [(int(i), int(c)) for i, c in fx[name + "_iou_keys"]]
    off = np.concatenate([[0], np.cumsum(np.prod(fx[name + "_iou_shape"], 1))])
    got = {k: v for k, v in E.ious.items() if len(v)}
    assert sorted(got) == sorted(keys)
    for j, k in enumerate(keys):
        assert got[k].shape == tuple(fx[name + "_iou_shape"][j])
        assert got[k].tobytes() == fx[name + "_iou_flat"][off[j]:off[j + 1]].tobytes()


@pytest.mark.parametrize("seed,n_img,n_cat", [(11, 300, 20), (12, 5000, 80)])
def test_device_equals_restatement(seed, n_img, n_cat):
    import cocoeval_np
    from sniper_b200 import cocoeval
    gt, res = F.synthetic_set(seed, n_img=n_img, n_cat=n_cat)
    cg = cocoeval.COCO(gt)
    cd = cg.loadRes(res)
    E = _evaluated(cg, cd, cocoeval.Params())
    p = E.params
    pk = E._pk
    r = cocoeval_np.match(pk, p.iouThrs, p.areaRng)
    for k in ('dt_flags', 'npig', 'gt_match'):
        dev = E._match[k].cpu().numpy().reshape(r[k].shape)
        assert dev.tobytes() == r[k].tobytes(), k
    prec, rec = cocoeval_np.accumulate(pk, r, p.maxDets, p.recThrs, pk['K'])
    assert E.eval['precision'].tobytes() == prec.tobytes()
    assert E.eval['recall'].tobytes() == rec.tobytes()
    assert (prec > 0).any() and (E._match['dt_flags'] & 1).any().item()


def test_evaluate_detections_end_to_end(fx, tmp_path):
    """coco.evaluate_detections on the fixture's synthetic set and detector output: the written rows are the reference
    writer's and the returned stats the reference's."""
    from sniper_b200 import coco
    gt = json.loads(bytes(fx["synth_gt_json"]).decode())
    (tmp_path / "data" / "annotations").mkdir(parents=True)
    (tmp_path / "data" / "annotations" / "instances_val2017.json").write_text(json.dumps(gt))
    imdb = coco.coco("val2017", str(tmp_path), str(tmp_path / "data"))
    nb, flat = fx["synth_boxes_n"], fx["synth_boxes"]
    all_boxes, k0 = [[None] * imdb.num_images for _ in range(nb.shape[0])], 0
    for k in range(nb.shape[0]):
        for i in range(imdb.num_images):
            all_boxes[k][i] = flat[k0:k0 + nb[k, i]]
            k0 += nb[k, i]
    stats = imdb.evaluate_detections(all_boxes)
    assert np.asarray(stats).tobytes() == fx["synth_stats"].tobytes()
    rows = json.load(open(tmp_path / "cache" / "results" / "detections_val2017_results.json"))
    assert np.array([r['bbox'] for r in rows]).tobytes() == fx["synth_rows_bbox"].tobytes()
    assert set(imdb.eval_times) >= {"write_s", "load_s", "pack_s", "match_s", "accumulate_s"}
    # a test split writes the file and does not evaluate
    (tmp_path / "data" / "annotations" / "image_info_test2017.json").write_text(json.dumps(gt))
    assert coco.coco("test2017", str(tmp_path), str(tmp_path / "data")).evaluate_detections(all_boxes) is None


def test_detection_wrapper_evaluates_with_an_imdb(tmp_path):
    from sniper_b200 import coco, iterator as IT, model, synth_batch
    from sniper_b200 import tester as TS
    cfg = IT.default_config()
    cfg.TEST.SCALES = [(96, 160), (192, 320), (288, 480)]
    cfg.TEST.BATCH_IMAGES = [2, 2, 1]
    cfg.TEST.VALID_RANGES = [(40, -1), (16, 90), (-1, 40)]
    cfg.TEST.CHIP_HYPERPARAMS = [(3, 0.3, 4), (3, 0.4, 5)]
    rng = np.random.RandomState(5)
    sizes = ((320, 240), (240, 320))
    cat_ids = [c for c in range(1, 91) if c not in (12, 26, 29, 30, 45, 66, 68, 69, 71, 83)]
    gt = dict(images=[dict(id=i + 1, width=w, height=h) for i, (w, h) in enumerate(sizes)],
              categories=[dict(id=c, name="c%d" % c, supercategory="s") for c in cat_ids],
              annotations=[dict(id=j + 1, image_id=1 + j % 2, category_id=cat_ids[j % 80],
                                bbox=[10.0 * j, 12.0, 40.0, 50.0], area=2000.0, iscrowd=0) for j in range(6)])
    (tmp_path / "data" / "annotations").mkdir(parents=True)
    (tmp_path / "data" / "annotations" / "instances_minival.json").write_text(json.dumps(gt))
    imdb = coco.coco("minival", str(tmp_path), str(tmp_path / "data"))
    assert imdb.num_classes == 81
    db = [dict(width=w, height=h, image_data=rng.randint(0, 256, (h, w, 3)).astype(np.uint8)) for (w, h) in sizes]
    mc = model.Cfg()
    mc.batch_images = 2
    net = model.SniperResNet101(mc, deform_offset_std=0.01)
    net.train_step(synth_batch.make_batch(2, seed=7, device="cuda"), lr=0.001)
    net.enable_autofocus(seed=3)
    all_boxes, stats = TS.imdb_detection_wrapper(net, cfg, db, imdb=imdb)
    assert np.asarray(stats['eval']).shape == (12,) and stats['eval_s'] > 0
    assert os.path.exists(tmp_path / "cache" / "results" / "detections_minival_results.json")
