"""PASCAL VOC evaluation without a device: the numpy restatement (oracle/voc_eval_np.py), the comp4 writer, gt_roidb and
the info string against the reference's own lib/dataset/pascal_voc.py / pascal_voc_eval.py
(tests/golden/voc_eval_ref.npz, oracle/run_ref_voc_eval.py), and the argument checks of csrc/voc_eval.cu.

The argument tests pass fabricated, never dereferenced device addresses (as test_cocoeval_cpu.py does): every call
violates one rule and must return from the check before any CUDA call; an empty input must return 0 without a launch."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", "oracle"))

import voc_eval_fixture as F  # noqa: E402
import voc_eval_np  # noqa: E402
from sniper_b200 import _lib, iterator, ops, pascal_voc  # noqa: E402


@pytest.fixture(scope="module")
def fx():
    return F.load()


@pytest.mark.parametrize("name", F.CASES)
def test_restatement_equals_reference(fx, name, tmp_path):
    dk = F.write_devkit(fx, name, str(tmp_path))
    det_box, det_pair, gt_box, gt_diff, gt_off, npos, det_off = F.device_inputs(fx, name, dk)
    flags = voc_eval_np.match(det_box, det_pair, gt_box, gt_diff, gt_off, (0.5, 0.7))
    for metric in ("07", "area"):
        rec, prec, ap = voc_eval_np.accumulate(flags, det_off, npos, metric == "07")
        for t, thr in enumerate(("0.5", "0.7")):
            k = "%s_%s_%s_" % (name, metric, thr)
            assert rec[t].tobytes() == fx[k + "rec"].tobytes(), k
            assert prec[t].tobytes() == fx[k + "prec"].tobytes(), k
            assert ap[t].tobytes() == fx[k + "ap"].tobytes(), k


def test_fixture_covers_the_edge_cases(fx):
    # a class with more than 128 recall changes (the pairwise sum recurses), NaN recall (npos = 0), ties in the text
    off, rec = fx["ties12_det_off"], fx["ties12_area_0.5_rec"]
    assert max(len(np.unique(rec[off[c]:off[c + 1]])) for c in range(20)) > 128
    assert np.isnan(fx["hand_area_0.5_ap"][2]) and fx["hand_07_0.5_ap"][2] == 0.0
    assert "nan" in str(fx["hand_info"])
    for name in ("ties07", "ties12"):
        off, si = fx[name + "_det_off"], fx[name + "_sorted_inds"]
        ties = 0
        for c in range(20):
            conf = np.array([float(l.split()[1]) for l in str(fx[name + "_text"][c]).splitlines()])
            ties += len(conf) - len(np.unique(conf))
            assert (np.diff(-conf[si[off[c]:off[c + 1]]]) >= 0).all()
        assert ties > 100


@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 127, 128, 129, 255, 256, 1000, 8191, 8193, 20001])
def test_pairwise_sum_is_np_sum(n):
    a = np.random.RandomState(n).rand(n) * 10.0 ** np.random.RandomState(n + 1).uniform(-6, 6, n)
    assert voc_eval_np.pairwise_sum(a).tobytes() == np.float64(np.sum(a)).tobytes()
    assert voc_eval_np.pairwise_sum(-np.zeros(n)).tobytes() == np.float64(np.sum(-np.zeros(n))).tobytes()


@pytest.mark.parametrize("name", F.CASES)
def test_host_voc_ap_equals_reference(fx, name):
    off = fx[name + "_det_off"]
    for metric in ("07", "area"):
        for thr in ("0.5", "0.7"):
            k = "%s_%s_%s_" % (name, metric, thr)
            for c in range(20):
                r, p = fx[k + "rec"][off[c]:off[c + 1]], fx[k + "prec"][off[c]:off[c + 1]]
                with np.errstate(invalid="ignore"):
                    ap = pascal_voc.voc_ap(r, p, metric == "07")
                assert np.float64(ap).tobytes() == fx[k + "ap"][c].tobytes()


@pytest.mark.parametrize("name", F.CASES)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_writer_text(fx, name, dtype, tmp_path):
    dk = F.write_devkit(fx, name, str(tmp_path))
    imdb = pascal_voc.PascalVOC(str(fx[name + "_year"]) + "_test", str(tmp_path), dk)
    ab = F.all_boxes(fx, name, dtype)
    os.makedirs(os.path.join(imdb.result_path, "results", "VOC" + imdb.year, "Main"))
    imdb.write_pascal_results(ab)
    for c, cls in enumerate(F.CLASSES):
        with open(imdb.get_result_file_template().format(cls)) as f:
            assert f.read() == str(fx[name + "_text"][c]), cls


@pytest.mark.parametrize("name", F.CASES)
def test_gt_roidb(fx, name, tmp_path):
    dk = F.write_devkit(fx, name, str(tmp_path))
    imdb = pascal_voc.PascalVOC(str(fx[name + "_year"]) + "_test", str(tmp_path), dk)
    assert imdb.name == "PASCALVOC_%s_test" % fx[name + "_year"] and imdb.num_classes == 21
    for roidb in (imdb.gt_roidb(), imdb.gt_roidb()):  # written, then read back from the cache
        assert [len(r["boxes"]) for r in roidb] == fx[name + "_roidb_n"].tolist()
        assert [os.path.relpath(r["image"], dk) for r in roidb] == fx[name + "_roidb_image"].tolist()
        assert all(type(r["height"]) is float and type(r["width"]) is float for r in roidb)
        assert np.array([[r["height"], r["width"]] for r in roidb]).tobytes() == fx[name + "_roidb_hw"].tobytes()
        assert [r["flipped"] for r in roidb] == fx[name + "_roidb_flipped"].tolist()
        for k in ("boxes", "gt_classes", "gt_overlaps", "max_classes", "max_overlaps"):
            got = np.concatenate([r[k] for r in roidb])
            ref = fx[name + "_roidb_" + k]
            assert got.dtype == ref.dtype and got.shape == ref.shape and got.tobytes() == ref.tobytes(), k


@pytest.mark.parametrize("name", F.CASES)
def test_info_string_from_reference_aps(fx, name, tmp_path, monkeypatch):
    dk = F.write_devkit(fx, name, str(tmp_path))
    year = str(fx[name + "_year"])
    imdb = pascal_voc.PascalVOC(year + "_test", str(tmp_path), dk)
    metric = "07" if int(year) < 2010 else "area"
    seen = {}

    def fake(detpath, annopath, imageset_file, classnames, annocache, ovthresh, use_07_metric, device, times):
        seen.update(classes=list(classnames), thr=tuple(ovthresh), use07=use_07_metric)
        return dict(ap=[list(fx["%s_%s_%s_ap" % (name, metric, t)]) for t in ("0.5", "0.7")])
    monkeypatch.setattr(pascal_voc, "voc_eval_classes", fake)
    info = imdb.evaluate_detections(F.all_boxes(fx, name))
    assert info == str(fx[name + "_info"])
    assert seen == dict(classes=F.CLASSES, thr=(0.5, 0.7), use07=metric == "07")
    assert "write_s" in imdb.eval_times


def test_default_config_pascal_voc():
    cfg = iterator.default_config(dataset="pascal_voc")
    assert cfg.dataset.NUM_CLASSES == 21
    assert cfg.network.PIXEL_MEANS == [103.939, 116.779, 123.68]
    assert cfg.network.RPN_FEAT_STRIDE == 16 and cfg.network.NUM_ANCHORS == 21
    t = cfg.TEST
    assert t.SCALES == [(1400, 2000), (800, 1280), (480, 512)] and t.BATCH_IMAGES == [2, 2, 4]
    assert t.VALID_RANGES == [(-1, 90), (32, 180), (75, -1)]
    assert t.AUTO_FOCUS is False and t.DO_PRUNING == [False, False, False]
    assert (t.MAX_PER_IMAGE, t.NMS, t.NMS_SIGMA) == (200, -1, 0.55)
    # the default is unchanged
    d = iterator.default_config()
    assert d.dataset.NUM_CLASSES == 81 and d.network.PIXEL_MEANS == [103.06, 115.90, 123.15]
    assert vars(iterator.default_config(dataset="coco").TEST) == vars(d.TEST)
    with pytest.raises(ValueError):
        iterator.default_config(dataset="imagenet")


# ---------------------------------------------------------------------------------------------------------------------
A_ = 0x7f0000100000
V = [A_ + 0x10000 * i for i in range(1, 24)]


def _h(a, t):
    a = np.ascontiguousarray(a, dtype=t)
    return a, a.ctypes.data


def _call(name, **kw):
    L = _lib.lib()
    return getattr(L, name)(*kw.values()), L.sniper_last_error().decode()


def _match_args(**over):
    pdo, pp = _h([0, 2, 3], np.int32)
    gto, gp = _h([0, 1, 3], np.int32)
    thr, tp = _h([0.5, 0.7], np.float64)
    kw = dict(det_box=V[0], pair_det_off=V[1], pair_det_pos=V[2], gt_box=V[3], gt_difficult=V[4], gt_off=V[5],
              pair_det_off_host=pp, gt_off_host=gp, P=2, thresholds=tp, T=2, flags=V[6], taken=V[7], stream=0)
    kw.update(over)
    return kw, (pdo, gto, thr)


def _acc_args(**over):
    off, op = _h([0, 2, 3], np.int32)
    t07, tp = _h(np.arange(0., 1.1, 0.1), np.float64)
    kw = dict(flags=V[0], det_off=V[1], npos=V[2], det_off_host=op, C=2, T=2, use_07_metric=0, thresholds_07=tp,
              n07=11, rec=V[3], prec=V[4], ap=V[5], terms=V[6], stream=0)
    kw.update(over)
    return kw, (off, t07)


def _bad(kwkeep, name, pattern):
    kw, keep = kwkeep
    rc, msg = _call(name, **kw)
    assert rc == -1, (name, kw)
    assert pattern in msg, (pattern, msg)


def test_match_refusals():
    n = "sniper_voc_match"
    _bad(_match_args(P=-1), n, "P (-1) must not be negative")
    _bad(_match_args(T=0), n, "T (0 overlap thresholds)")
    _bad(_match_args(T=17), n, "T (17 overlap thresholds)")
    _bad(_match_args(thresholds=0), n, "thresholds (host) must not be null")
    _bad(_match_args(gt_off_host=0), n, "host offsets")
    bad, bp = _h([0, 2, 1], np.int32)
    _bad(_match_args(pair_det_off_host=bp), n, "pair_det_off must start at 0 and not decrease")
    bad2, bp2 = _h([1, 2, 3], np.int32)
    _bad(_match_args(gt_off_host=bp2), n, "gt_off must start at 0 and not decrease")
    _bad(_match_args(gt_off=0), n, "pair_det_off / gt_off must not be null")
    _bad(_match_args(pair_det_pos=0), n, "det_box / pair_det_pos / flags must not be null")
    _bad(_match_args(taken=0), n, "gt_box / gt_difficult / taken must not be null")
    assert _call(n, **_match_args(P=0)[0])[0] == 0
    z, zp = _h([0, 0, 0], np.int32)
    assert _call(n, **_match_args(pair_det_off_host=zp)[0])[0] == 0  # no detections: nothing to launch


def test_accumulate_refusals():
    n = "sniper_voc_accumulate"
    _bad(_acc_args(C=-1), n, "C (-1) must not be negative")
    _bad(_acc_args(T=0), n, "T (0 overlap thresholds)")
    _bad(_acc_args(use_07_metric=2), n, "use_07_metric (2) must be 0 or 1")
    _bad(_acc_args(use_07_metric=1, n07=0), n, "n07 (0 recall thresholds)")
    _bad(_acc_args(use_07_metric=1, n07=33), n, "n07 (33 recall thresholds)")
    _bad(_acc_args(use_07_metric=1, thresholds_07=0), n, "thresholds_07 (host) must not be null")
    _bad(_acc_args(det_off_host=0), n, "host offsets")
    bad, bp = _h([0, 3, 2], np.int32)
    _bad(_acc_args(det_off_host=bp), n, "det_off must start at 0 and not decrease")
    _bad(_acc_args(npos=0), n, "det_off / npos / ap must not be null")
    _bad(_acc_args(prec=0), n, "flags / rec / prec must not be null")
    _bad(_acc_args(terms=0), n, "terms must not be null for the area metric")
    assert _call(n, **_acc_args(C=0)[0])[0] == 0


def test_ops_refuse_bad_inputs_before_launch():
    box = torch.zeros(3, 4, dtype=torch.float64)
    gt = torch.zeros(2, 4, dtype=torch.float64)
    diff = torch.zeros(2, dtype=torch.uint8)
    with pytest.raises(ValueError, match="pair index is outside"):
        ops.voc_match(box, [0, 1, 4], gt, diff, [0, 1, 1, 2, 2], (0.5,))
    with pytest.raises(ValueError, match="det_box must be"):
        ops.voc_match(box[:2], [0, 1, 2], gt, diff, [0, 1, 1, 2, 2], (0.5,))
    with pytest.raises(ValueError, match="gt_box"):
        ops.voc_match(box, [0, 1, 2], gt[:1], diff, [0, 1, 1, 2, 2], (0.5,))
    with pytest.raises(ValueError, match="det_off ends at 2"):
        ops.voc_accumulate(torch.zeros(2, 3, dtype=torch.uint8), [0, 1, 2], torch.zeros(2, dtype=torch.int32), False)
