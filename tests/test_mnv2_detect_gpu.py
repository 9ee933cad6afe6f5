"""The MobileNetV2 detector through the multi-scale inference pyramid on the device: stride-32 canvases, both detection
backends and both soft-NMS backends, COCO evaluation of a network loaded from a `fit` checkpoint, and one inference pass
at each shipped test scale's largest canvas."""
import itertools
import json

import numpy as np
import pytest
import torch

from sniper_b200 import callback, checkpoint, coco, model_mnv2, synth_batch, trainer
from sniper_b200 import iterator as IT
from sniper_b200 import tester as TS

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _small_cfg():
    cfg = IT.default_config(network="mobilenetv2")
    cfg.TEST.SCALES = [(288, 480), (192, 320), (96, 160)]      # same structure as (1400,2000) / (800,1280) / (480,512)
    cfg.TEST.BATCH_IMAGES = [1, 2, 2]
    cfg.TEST.VALID_RANGES = [(-1, 40), (16, 90), (40, -1)]
    return cfg


def _net(seed=3, train=True):
    mc = model_mnv2.MCfg()
    mc.batch_images, mc.bf16 = 2, True
    net = model_mnv2.SniperMobileNetV2(mc, device=DEV, seed=seed)
    if train:                                                   # non-trivial moving statistics
        net.train_step(synth_batch.make_batch(2, seed=7, device=DEV, A=mc.num_anchors, stride=mc.feat_stride), lr=0.001)
    return net


def _images(sizes, seed=2):
    rng = np.random.RandomState(seed)
    return [dict(width=W, height=H, image_data=rng.randint(0, 256, (H, W, 3)).astype(np.uint8)) for (W, H) in sizes]


def _check_inside(all_boxes, db):
    n = 0
    for j in range(1, 81):
        for i, r in enumerate(db):
            d = all_boxes[j][i]
            assert d.ndim == 2 and d.shape[1] == 5 and np.isfinite(d).all()
            assert (d[:, :4] >= 0).all() and (d[:, 0] <= d[:, 2]).all() and (d[:, 1] <= d[:, 3]).all()
            assert (d[:, [0, 2]] <= r['width']).all() and (d[:, [1, 3]] <= r['height']).all()
            n += len(d)
    return n


def test_mobilenet_pyramid_backends_agree():
    """Three images of different orientations through the three-scale pyramid: the device detection backend keeps the
    host backend's rows (its float32 box decoding differs in the last bits), device and host soft-NMS give the same
    detections, and no parameter changes."""
    cfg = _small_cfg()
    db = _images(((320, 240), (240, 320), (300, 200)))
    net = _net()
    w0 = net.P.w.cpu().numpy().tobytes()
    canv = [b['data'].shape[2:] for b in TS.MNIteratorTestAutoFocus(
        [dict(r, inference_crops=np.array([[0, 0, r['width'], r['height']]])) for r in db], cfg, cfg.TEST.SCALES[0],
        batch_size=1)]
    assert all(h % 32 == 0 and w % 256 == 0 for h, w in canv)
    boxes_h, stats_h = TS.imdb_detection_wrapper(net, cfg, db, detect_backend="host")
    boxes_d, stats_d = TS.imdb_detection_wrapper(net, cfg, db, detect_backend="device")
    boxes_dh, _ = TS.imdb_detection_wrapper(net, cfg, db, detect_backend="device", nms_backend="host")
    torch.cuda.synchronize()
    assert net.P.w.cpu().numpy().tobytes() == w0
    assert [s['chips'] for s in stats_d['scales']] == [s['chips'] for s in stats_h['scales']] == [3, 3, 3]
    pre = [s['detections_pre_nms'] for s in stats_d['scales']]
    assert min(pre) > 0
    n, worst_box, worst_score = 0, 0.0, 0.0
    for j in range(1, 81):
        for i in range(3):
            a, b, c = boxes_d[j][i], boxes_h[j][i], boxes_dh[j][i]
            assert a.shape == b.shape == c.shape and a.dtype == b.dtype == np.float32
            assert np.array_equal(a[:, :4], c[:, :4]) and np.abs(a[:, 4] - c[:, 4]).max(initial=0) < 1e-6
            if len(a):
                worst_box = max(worst_box, float(np.abs(a[:, :4].astype(np.float64) - b[:, :4]).max()))
                worst_score = max(worst_score, float(np.abs(a[:, 4].astype(np.float64) - b[:, 4]).max()))
            n += len(a)
    print("detections before the NMS per scale:", pre, "; %d final; device vs host detection backend: boxes within "
          "%.3g px, scores within %.3g" % (n, worst_box, worst_score))
    assert n > 0 and worst_box < 1e-3 and worst_score < 1e-5
    assert _check_inside(boxes_d, db) == n == _check_inside(boxes_h, db)
    assert n <= 3 * cfg.TEST.MAX_PER_IMAGE + 80 * 3


class _Steps(object):
    """The first `n` raw batches of an iterator as one epoch (Trainer.fit's iterator protocol)."""

    def __init__(self, it, n):
        self.it, self.n = it, n

    def __iter__(self):
        return itertools.islice(self.it, self.n)

    def reset(self):
        self.it.reset()


def test_coco_evaluation_from_a_fit_checkpoint(tmp_path):
    """Two fit steps, the epoch-end checkpoint, main_test.py's loading (`*_test` tensors over the training ones) into a
    fresh net, then the pyramid with a COCO imdb."""
    np.random.seed(5)
    tcfg = IT.default_config(network="mobilenetv2")
    B = 2
    it = IT.MNIteratorE2E(IT.synthetic_roidb(2, seed=6, n_gt=(2, 10)), tcfg, batch_size=B, n_buffers=4)
    net = _net(seed=3, train=False)
    tr = trainer.Trainer(net.cfg, device=DEV, net=net, scheduler=None)
    prefix = str(tmp_path / "mnv2")
    tr.fit(_Steps(it, 2), IT.InputStage(tcfg, DEV, B), 1, epoch_end_callback=callback.module_checkpoint(tr, prefix))
    assert tr.num_update == 2
    arg, aux = checkpoint.load_param(prefix, 1, process=True)
    raw, _ = checkpoint.load_param(prefix, 1)
    stds = np.array(checkpoint.BBOX_STDS_TEST, np.float32)
    assert np.array_equal(arg["bbox_pred_weight"], raw["bbox_pred_weight_test"])
    assert np.array_equal(arg["bbox_pred_weight"], (raw["bbox_pred_weight"].T * stds).T)
    fresh = _net(seed=9, train=False)
    fresh.load_reference(arg, aux)
    earg, eaux = fresh.export_reference()
    assert set(earg) == set(arg) and set(eaux) == set(aux)
    assert all(earg[k].tobytes() == arg[k].tobytes() for k in arg) and all(eaux[k].tobytes() == aux[k].tobytes() for k in aux)

    sizes = ((320, 240), (240, 320), (300, 200))
    cat_ids = [c for c in range(1, 91) if c not in (12, 26, 29, 30, 45, 66, 68, 69, 71, 83)]
    gt = dict(images=[dict(id=i + 1, width=w, height=h) for i, (w, h) in enumerate(sizes)],
              categories=[dict(id=c, name="c%d" % c, supercategory="s") for c in cat_ids],
              annotations=[dict(id=j + 1, image_id=1 + j % 3, category_id=cat_ids[j % 80],
                                bbox=[10.0 * j, 12.0, 40.0, 50.0], area=2000.0, iscrowd=0) for j in range(9)])
    (tmp_path / "data" / "annotations").mkdir(parents=True)
    (tmp_path / "data" / "annotations" / "instances_minival.json").write_text(json.dumps(gt))
    imdb = coco.coco("minival", str(tmp_path), str(tmp_path / "data"))
    db = _images(sizes, seed=4)
    all_boxes, stats = TS.imdb_detection_wrapper(fresh, _small_cfg(), db, imdb=imdb, detect_backend="device")
    ev = np.asarray(stats['eval'], np.float64)
    print("COCO stats of the two-step network:", ev.tolist())
    assert ev.shape == (12,) and all(np.isfinite(v) and (v == -1 or 0 <= v <= 1) for v in ev)
    assert _check_inside(all_boxes, db) > 0


@pytest.mark.parametrize("B, H, W", [(2, 1408, 2048), (2, 832, 1280), (4, 512, 512)])
def test_forward_inference_at_the_largest_test_canvases(B, H, W):
    """The largest canvas of each shipped test scale (TEST.SCALES (1400,2000) / (800,1280) / (480,512) with their
    batch sizes): a 44 x 64 last map at the first."""
    net = _net(seed=5)
    assert TS._canvas_size(H, W, 32) == (H, W)
    g = torch.Generator(device=DEV).manual_seed(B * H)
    data = torch.randn(B, 3, H, W, device=DEV, generator=g) * 60.0
    im_info = torch.tensor([[H, W, 1.0]] * B, device=DEV)
    rois, scores, cls_prob, bbox_pred = net.forward_inference(data, im_info)
    torch.cuda.synchronize()
    assert rois.shape == (B * 300, 5) and cls_prob.shape == (B * 300, 81) and bbox_pred.shape == (B * 300, 4)
    r = rois.cpu().numpy()
    assert [int((r[:, 0] == b).sum()) for b in range(B)] == [300] * B
    assert (r[:, 1:] >= 0).all() and (r[:, [1, 3]] <= W - 1).all() and (r[:, [2, 4]] <= H - 1).all()
    p = cls_prob.double()
    assert torch.isfinite(p).all() and torch.isfinite(bbox_pred).all() and torch.isfinite(scores).all()
    assert float((p.sum(1) - 1).abs().max()) < 1e-5
