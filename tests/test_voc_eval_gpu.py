"""PASCAL VOC evaluation on the device (csrc/voc_eval.cu through sniper_b200.pascal_voc): bit for bit against the
reference's own voc_eval on the fixture cases (tests/golden/voc_eval_ref.npz), fed the order the reference's
np.argsort recorded; against the numpy restatement (oracle/voc_eval_np.py) on seeded tied sets up to VOC2007 test's
shape, with the order np.argsort gives in this process; then the imdb and the test wrapper end to end.  NaN values only
have to sit where the reference's do (voc_eval_fixture.same)."""
import os
import re
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", "oracle"))

import voc_eval_fixture as F  # noqa: E402
import voc_eval_np  # noqa: E402
from sniper_b200 import ops, pascal_voc  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def fx():
    return F.load()


def _device(det_box, det_pair, gt_box, gt_diff, gt_off, npos, det_off, use07, thr=(0.5, 0.7)):
    d = torch.device(DEV)
    flags = ops.voc_match(torch.from_numpy(np.ascontiguousarray(det_box)).to(d), det_pair,
                          torch.from_numpy(gt_box).to(d), torch.from_numpy(gt_diff).to(d), gt_off, thr)
    rec, prec, ap = ops.voc_accumulate(flags, det_off, torch.from_numpy(npos).to(d), use07)
    return flags.cpu().numpy(), rec.cpu().numpy(), prec.cpu().numpy(), ap.cpu().numpy()


@pytest.mark.parametrize("name", F.CASES)
def test_device_equals_reference(fx, name, tmp_path):
    dk = F.write_devkit(fx, name, str(tmp_path))
    inputs = F.device_inputs(fx, name, dk)
    for metric in ("07", "area"):
        _, rec, prec, ap = _device(*inputs, use07=metric == "07")
        for t, thr in enumerate(("0.5", "0.7")):
            k = "%s_%s_%s_" % (name, metric, thr)
            assert F.same(rec[t], fx[k + "rec"]), k
            assert F.same(prec[t], fx[k + "prec"]), k
            assert F.same(ap[t], fx[k + "ap"]), k


def _tied_set(seed, n_img, n_cls, per_img, det_per_img):
    """VOC-shaped arrays: ~per_img objects per image (15% difficult), det_per_img detections per image, most near a GT,
    scores with 3 decimals (heavy ties), boxes with 1; the per-class order is np.argsort(-confidence)."""
    rng = np.random.RandomState(seed)
    n_obj = rng.poisson(per_img, n_img)
    img = np.repeat(np.arange(n_img), n_obj)
    G = img.size
    cls = rng.randint(n_cls, size=G)
    wh = rng.randint(8, 250, (G, 2))
    xy = rng.randint(1, 250, (G, 2))
    gbox = np.concatenate([xy, xy + wh], 1).astype(np.float64)
    diff = (rng.rand(G) < 0.15)
    key = cls * n_img + img
    order = np.argsort(key, kind="stable")
    gt_off = np.zeros(n_cls * n_img + 1, np.int32)
    np.cumsum(np.bincount(key, minlength=n_cls * n_img), out=gt_off[1:])
    npos = np.bincount(cls[~diff], minlength=n_cls).astype(np.int32)
    N = n_img * det_per_img
    dimg = np.repeat(np.arange(n_img), det_per_img)
    near = (rng.rand(N) < 0.6) & (n_obj[dimg] > 0)
    g = np.minimum(np.cumsum(np.concatenate([[0], n_obj]))[dimg] + (rng.rand(N) * np.maximum(n_obj[dimg], 1)).astype(int),
                   G - 1)
    dcls = np.where(near, cls[g], rng.randint(n_cls, size=N))
    dbox = np.where(near[:, None], gbox[g] + rng.randn(N, 4) * rng.choice([0.5, 4.0, 15.0], (N, 1)),
                    rng.uniform(0, 300, (N, 4)))
    dbox[:, 2:] = np.where(near[:, None], dbox[:, 2:], dbox[:, :2] + rng.uniform(0, 120, (N, 2)))
    dbox = np.round(dbox, 1)
    conf = np.round(rng.rand(N), 3)
    boxes, pairs, det_off = [], [], [0]
    for c in range(n_cls):
        sel = np.flatnonzero(dcls == c)
        s = np.argsort(-conf[sel])
        boxes.append(dbox[sel][s])
        pairs.append(c * n_img + dimg[sel][s])
        det_off.append(det_off[-1] + sel.size)
    return (np.concatenate(boxes), np.concatenate(pairs), gbox[order], diff[order].astype(np.uint8), gt_off, npos,
            np.asarray(det_off, np.int32))


@pytest.mark.parametrize("seed,n_img,per_img,det_per_img", [(21, 40, 3, 30), (22, 600, 3, 200),
                                                             (23, 4952, 3, 200)])
def test_device_equals_restatement(seed, n_img, per_img, det_per_img):
    inputs = _tied_set(seed, n_img, 20, per_img, det_per_img)
    det_box, det_pair, gt_box, gt_diff, gt_off, npos, det_off = inputs
    ref_flags = voc_eval_np.match(det_box, det_pair, gt_box, gt_diff, gt_off, (0.5, 0.7))
    for use07 in (True, False):
        flags, rec, prec, ap = _device(*inputs, use07=use07)
        assert flags.tobytes() == ref_flags.tobytes()
        r_rec, r_prec, r_ap = voc_eval_np.accumulate(ref_flags, det_off, npos, use07)
        assert rec.tobytes() == r_rec.tobytes() and prec.tobytes() == r_prec.tobytes()
        assert ap.tobytes() == r_ap.tobytes(), (ap, r_ap)
    assert (ref_flags == 1).any() and (ref_flags == 0).any() and (ap > 0).any()


@pytest.mark.parametrize("name", F.CASES)
def test_evaluate_detections_end_to_end(fx, name, tmp_path):
    """PascalVOC.evaluate_detections on the case's devkit: the files it writes are the reference's and its info string
    is the reference's, byte for byte; voc_eval of one class equals the batched evaluation."""
    dk = F.write_devkit(fx, name, str(tmp_path))
    imdb = pascal_voc.PascalVOC(str(fx[name + "_year"]) + "_test", str(tmp_path), dk, device=DEV)
    info = imdb.evaluate_detections(F.all_boxes(fx, name))
    assert info == str(fx[name + "_info"])
    assert set(imdb.eval_times) >= {"write_s", "parse_s", "sort_s", "device_s"}
    tmpl = imdb.get_result_file_template()
    assert all(open(tmpl.format(c)).read() == str(fx[name + "_text"][k]) for k, c in enumerate(F.CLASSES))
    annopath = os.path.join(imdb.data_path, "Annotations", "{0!s}.xml")
    imageset = os.path.join(imdb.data_path, "ImageSets", "Main", "test.txt")
    cache = os.path.join(imdb.cache_path, imdb.name + "_annotations.pkl")
    off = fx[name + "_det_off"]
    for c in (0, 2, 14):
        rec, prec, ap = pascal_voc.voc_eval(tmpl.format(F.CLASSES[c]), annopath, imageset, F.CLASSES[c], cache,
                                            ovthresh=0.7, use_07_metric=False, device=DEV)
        k = name + "_area_0.7_"
        assert F.same(rec, fx[k + "rec"][off[c]:off[c + 1]]) and F.same(prec, fx[k + "prec"][off[c]:off[c + 1]])
        assert F.same(ap, fx[k + "ap"][c])


def test_detection_wrapper_evaluates_a_21_class_network(fx, tmp_path):
    """A 21-class SniperResNet101 trained for two steps on a VOC devkit's gt_roidb (seeded pixels), then the test
    wrapper with the VOC imdb: the info string is well formed and its APs are the restatement's on the files written."""
    from sniper_b200 import iterator as IT
    from sniper_b200 import model, trainer
    from sniper_b200 import tester as TS
    import itertools
    dk = F.write_devkit(fx, "hand", str(tmp_path))
    voc = pascal_voc.PascalVOC("2012_test", str(tmp_path), dk, device=DEV)
    roidb = voc.gt_roidb()

    def load(path):
        r = roidb[[x['image'] for x in roidb].index(path)]
        rng = np.random.RandomState(int(os.path.basename(path)[:-4]))
        return rng.randint(0, 256, (int(r['height']), int(r['width']), 3)).astype(np.uint8)

    tcfg = IT.default_config(neg=False, dataset="pascal_voc")
    train_db = [dict(r, boxes=r['boxes'].astype(np.float32), max_overlaps=r['max_overlaps'], width=int(r['width']),
                     height=int(r['height'])) for r in roidb if len(r['boxes'])]
    np.random.seed(5)
    it = IT.MNIteratorE2E(train_db, tcfg, batch_size=2, image_loader=load, n_buffers=4)
    mc = model.Cfg()
    mc.num_classes, mc.batch_images = 21, 2
    net = model.SniperResNet101(mc, deform_offset_std=0.01)
    tr = trainer.Trainer(net.cfg, device=DEV, net=net, scheduler=None)

    class Steps(object):
        def __iter__(self):
            return itertools.islice(it, 2)

        def reset(self):
            it.reset()
    tr.fit(Steps(), IT.InputStage(tcfg, DEV, 2), 1)
    assert tr.num_update == 2
    cfg = IT.default_config(dataset="pascal_voc")
    cfg.TEST.SCALES = [(288, 480), (192, 320), (96, 160)]
    cfg.TEST.BATCH_IMAGES = [2, 2, 2]
    cfg.TEST.VALID_RANGES = [(-1, 40), (16, 90), (40, -1)]
    db = [dict(width=int(r['width']), height=int(r['height']), image_data=load(r['image'])) for r in roidb]
    all_boxes, stats = TS.imdb_detection_wrapper(net, cfg, db, num_classes=21, imdb=voc)
    assert len(all_boxes) == 21 and sum(len(all_boxes[j][i]) for j in range(1, 21) for i in range(len(db))) > 0
    info = stats['eval']
    lines = info.split('\n')
    assert lines[0] == 'VOC07 metric? No' and len(lines) == 1 + 20 + 1 + 1 + 20 + 1
    pat = re.compile(r'^AP for (\w+) = (nan|\d\.\d{4})$')
    assert [pat.match(l).group(1) for l in lines[1:21] + lines[23:43]] == F.CLASSES * 2
    assert re.match(r'^Mean AP@0\.5 = (nan|\d\.\d{4})$', lines[21]) and lines[22] == ''
    assert re.match(r'^Mean AP@0\.7 = (nan|\d\.\d{4})$', lines[43])
    # the restatement on the written files, in the host's order
    images = list(voc.image_set_index)
    recs = {n: pascal_voc.parse_voc_rec(os.path.join(voc.data_path, 'Annotations', n + '.xml')) for n in images}
    gt_box, gt_diff, gt_off, npos = pascal_voc.gt_csr(recs, images, F.CLASSES)
    boxes, pairs, det_off = [], [], [0]
    for c, cls in enumerate(F.CLASSES):
        ids, conf, bbox = pascal_voc.read_detections(voc.get_result_file_template().format(cls))
        s = np.argsort(-conf)
        boxes.append(bbox[s].reshape(-1, 4))
        pairs.append(c * len(images) + np.array([images.index(x) for x in ids], np.int64)[s])
        det_off.append(det_off[-1] + len(s))
    flags = voc_eval_np.match(np.concatenate(boxes), np.concatenate(pairs), gt_box, gt_diff, gt_off, (0.5, 0.7))
    _, _, ap = voc_eval_np.accumulate(flags, np.asarray(det_off), npos, False)
    assert info == pascal_voc.info_string([list(zip(F.CLASSES, ap[0])), list(zip(F.CLASSES, ap[1]))], False)
    print(info)
