"""Training from an image set on disk (tools/train_e2e.py) on the device: a synthetic VOCdevkit with JPEG files read by
host.imread -> the roidb of 2007_trainval + 2012_trainval (flipped, merged, filtered, targets) -> two epochs of
Trainer.fit of the 21-class ResNet-101 (TF32 and bf16 backbone), every Speedometer window checked against the float64
restatement -> per-epoch checkpoints read back -> evaluation on 2007_test with the VOC imdb.  Then RPN proposals of both
training sets from the trained network (imdb_proposal_extraction_wrapper) feed one epoch with negative chips, so the
rpn_roidb branch and its device NMS run; and the iterator's chips of a flipped entry reach the network mirrored."""
import os
import re
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", "tools"))

import test_fit_gpu as FIT  # noqa: E402
import train_data_fixture as TD  # noqa: E402
import train_e2e as E  # noqa: E402
from sniper_b200 import callback, checkpoint, host, load_data, tester  # noqa: E402
from sniper_b200 import iterator as IT  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B = 2


class _Checked(object):
    """Every step: finite losses; every Speedometer window: the metrics equal the float64 restatement
    (test_fit_gpu._Window, bound to the trainer fit runs)."""

    def __init__(self):
        self.sp = callback.Speedometer(B, 2)
        self.win = None
        self.steps = 0

    def __call__(self, p):
        tr = p.locals["self"]
        if self.win is None:
            self.win = FIT._Window(tr, self.sp)
        self.win(p)
        assert torch.isfinite(tr.out["losses"]).all(), tr.out["losses"]
        self.sp(p)
        self.steps += 1


def _argv(root, dk, prefix, *extra):
    return ["--dataset", "PascalVOC", "--image-set", "2007_trainval+2012_trainval", "--root-path", root,
            "--dataset-path", dk, "--batch-size", str(B), "--display", "2", "--prefix", prefix,
            "--device", DEV] + list(extra)


def _info_ok(info):
    lines = info.split("\n")
    assert lines[0] == "VOC07 metric? Y" and len(lines) == 1 + 20 + 1 + 1 + 20 + 1
    pat = re.compile(r"^AP for (\w+) = (nan|\d\.\d{4})$")
    assert [pat.match(l).group(1) for l in lines[1:21] + lines[23:43]] == TD.VOC_CLASSES * 2
    assert re.match(r"^Mean AP@0\.5 = (nan|\d\.\d{4})$", lines[21])


@pytest.mark.parametrize("bf16", [False, True], ids=["tf32", "bf16"])
def test_train_checkpoint_evaluate_from_jpeg(tmp_path, bf16):
    np.random.seed(7)
    root = str(tmp_path)
    dk, listing = TD.write_voc(root)
    prefix = os.path.join(root, "out", "voc")
    chk = _Checked()
    argv = _argv(root, dk, prefix, "--epochs", "2", "--test-image-set", "2007_test", *(["--bf16"] if bf16 else []))
    out = E.main(argv, batch_end_callback=chk)
    t = out["times"]
    assert t["entries"] == 12 and t["entries_kept"] == 8           # the last image of each set has only difficult GT
    assert all(t[k] >= 0 for k in ("gt_s", "rpn_s", "flip_s", "filter_s", "targets_s")) and t["imread_s_per_image"] > 0
    tr = out["trainer"]
    assert chk.steps > 0 and chk.win.checked >= 2 and tr.num_update == chk.steps
    # the checkpoints of both epochs, read back: the last one holds the trained weights and statistics
    for ep in (1, 2):
        assert os.path.isfile("%s-%04d.params" % (prefix, ep)) and os.path.isfile("%s-%04d.states" % (prefix, ep))
    arg, aux = checkpoint.load_param(prefix, 2)
    want_arg, want_aux = tr.net.export_reference()
    assert all(arg[k].tobytes() == v.tobytes() for k, v in want_arg.items())
    assert all(aux[k].tobytes() == v.tobytes() for k, v in want_aux.items())
    net = E.make_net(E.parse_args(argv), 21, B, DEV)
    net.load_reference(arg, aux)
    got_arg, _ = net.export_reference()
    assert all(got_arg[k].tobytes() == v.tobytes() for k, v in want_arg.items())
    # the evaluation on 2007_test
    all_boxes, stats = out["all_boxes"], out["stats"]
    assert len(all_boxes) == 21 and all(len(c) == len(listing["2007_test"]) for c in all_boxes)
    _info_ok(stats["eval"])
    if bf16:
        return
    # RPN proposals of both training sets from the trained network, then one epoch with negative chips
    pp = os.path.join(root, "proposals")
    cfg = E.config_for(E.parse_args(argv))
    arg, aux = checkpoint.load_param(prefix, 2, process=True)
    rpn_net = E.make_net(E.parse_args(argv), 21, 1, DEV)
    rpn_net.load_reference(arg, aux, allow_missing=True)
    for s in ("2007_trainval", "2012_trainval"):
        voc = load_data.DATASETS["PascalVOC"](s, root, dk, device=DEV)
        db = [dict(image=r["image"], width=int(r["width"]), height=int(r["height"])) for r in voc.gt_roidb()]
        cfg.dataset.test_image_set = s
        props, _ = tester.imdb_proposal_extraction_wrapper(rpn_net, cfg, db, pp, image_loader=host.imread)
        assert os.path.isfile(os.path.join(pp, "PASCALVOC_%s_rpn.pkl" % s)) and sum(len(p) for p in props) > 0
    del rpn_net
    chk = _Checked()
    neg_prefix = os.path.join(root, "out", "voc_neg")
    out = E.main(_argv(root, dk, neg_prefix, "--epochs", "1", "--proposal-path", pp), batch_end_callback=chk)
    assert out["times"]["rpn_s"] > 0 and chk.steps > 0 and chk.win.checked >= 1
    assert os.path.isfile(os.path.join(pp, "PASCALVOC_2007_trainval_rpn_after_nms.pkl"))
    assert os.path.isfile("%s-0001.params" % neg_prefix)


def test_flipped_entry_reaches_the_network_mirrored(tmp_path):
    """The input stage's chip of a flipped entry read from its JPEG equals, bit for bit, the chip of the same entry with
    its pixels mirrored in memory and flipped=False."""
    dk, _ = TD.write_voc(str(tmp_path), sets=(("2007", "trainval", 2),), size=(400, 300), empty_last=False)
    cfg = IT.default_config(neg=False, dataset="pascal_voc")
    r = load_data.load_proposal_roidb("PascalVOC", "2007_trainval", str(tmp_path), dk, flip=True, only_gt=True,
                                      device=DEV)
    stage = IT.InputStage(cfg, DEV, 1)
    for e in r[2:]:
        twin = dict(e, flipped=False, image_data=np.ascontiguousarray(host.imread(e["image"])[:, ::-1]))
        data = []
        for entry in (dict(e), twin):
            np.random.seed(4)
            host.srand(4)
            it = IT.MNIteratorE2E([entry], cfg, batch_size=1, image_loader=host.imread, n_buffers=3)
            data.append(stage.run(it._get_batch(), subsample=False)["data"].clone())
        torch.cuda.synchronize()
        assert data[0].abs().sum() > 0 and torch.equal(data[0], data[1])
