"""The training metrics without a device: the float64 restatement against the reference's own metric classes (the
fixture of oracle/run_ref_metric.py), the names and order of the composite main_train.py builds, the value rules of
`get()`, and every argument refusal of `sniper_train_metric_accum` (fabricated, never dereferenced pointers: each call
violates one rule and returns from its check before any CUDA call)."""
import math
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import train_metric_np as T  # noqa: E402
from sniper_b200 import _lib, metric  # noqa: E402

FIX = os.path.join(ROOT, "tests", "golden", "train_metric_ref.npz")
CASES = ("resnet101_af", "mobilenetv2", "ignored")
LOGLOSS = (1, 4, 7)


def case(z, name):
    g = lambda k: z[name + "/" + k]
    af = (name + "/af_prob") in z
    return dict(rpn_prob=g("rpn_prob"), rpn_label=g("rpn_label"), A=int(g("A")), cls_prob=g("cls_prob"),
                cls_label=g("cls_label"), rpn_l1=g("rpn_l1"), rcnn_l1=g("rcnn_l1"),
                af_prob=g("af_prob") if af else None, af_label=g("af_label") if af else None)


@pytest.mark.parametrize("name", CASES)
def test_restatement_equals_the_reference_classes(name):
    """Counts, hit counts and L1 sums byte-equal.  The reference takes log(p + 1e-14) in float32 (one rounding per
    term, < 2^-24 relative) and sums the terms with numpy's float32 pairwise summation (< (8 + log2 n) roundings of
    2^-24 relative to the sum of the positive terms); the restatement does both in float64.  So the two log-loss sums
    differ by at most (10 + log2 n) * 2^-24 of their value."""
    z = np.load(FIX)
    num, s = T.step(**case(z, name))
    ref_sum, ref_num = z[name + "/sum_metric"], z[name + "/num_inst"]
    af = (name + "/af_prob") in z
    slots = range(8) if af else range(6)
    assert np.array_equal(num[list(slots)], ref_num[list(slots)])
    for k in slots:
        if k in LOGLOSS:
            n = max(int(num[k]), 1)
            bound = (10 + math.log2(n)) * 2.0 ** -24 * abs(ref_sum[k])
            assert abs(s[k] - ref_sum[k]) <= bound, (k, s[k], ref_sum[k])
        else:
            assert s[k] == ref_sum[k], (k, s[k], ref_sum[k])


def test_fixture_holds_the_edge_cases():
    z = np.load(FIX)
    p = T.two_way_rows(z["resnet101_af/rpn_prob"], 21)
    assert ((p[:, 0] == 0.5) & (p[:, 1] == 0.5)).any() and (p == 0).any()
    c = z["resnet101_af/cls_prob"]
    assert (np.sort(c, 1)[:, -1] == np.sort(c, 1)[:, -2]).any()
    assert (z["ignored/rpn_label"] == -1).all() and (z["ignored/cls_label"] == -1).all()
    assert z["mobilenetv2/rpn_prob"].shape == (2, 16, 16, 30) and z["resnet101_af/af_prob"].shape[1:] == (32, 32, 2)
    assert c.shape[1] == 81


def test_composite_names_and_order_follow_main_train():
    """main_train.py:104-128: RPNAcc, RPNLogLoss, RPNL1Loss, RCNNAcc, RCNNLogLoss, RCNNL1LossCRCNN, then (AUTO_FOCUS)
    AutoFocusAcc, AutoFocusLogLoss."""
    base = ["RPNAcc", "RPNLogLoss", "RPNL1Loss", "RCNNAcc", "RCNNLogLoss", "RCNNL1LossCRCNN"]
    for af, names in ((False, base), (True, base + ["AutoFocusAcc", "AutoFocusLogLoss"])):
        m = metric.default_metrics(af)
        m.bind(metric.MetricAccumulator("cpu"))
        assert [k for k, _ in m.get_name_value()] == names


def test_get_divides_and_gives_nan_without_instances():
    acc = metric.MetricAccumulator("cpu")
    m = metric.default_metrics(True)
    m.bind(acc)
    acc.buf[:8] = torch.tensor([4, 4, 4, 2, 2, 2, 0, 0])
    acc.buf[8:16] = torch.tensor([3, 0, 0, 1, 0, 0, 0, 0])
    acc.buf[16:].view(torch.float64).copy_(torch.tensor([0, 2.0, 1.0, 0, 3.0, 5.0, 0, 0], dtype=torch.float64))
    v = dict(m.get_name_value())
    assert v["RPNAcc"] == 0.75 and v["RPNLogLoss"] == 0.5 and v["RPNL1Loss"] == 0.25
    assert v["RCNNAcc"] == 0.5 and v["RCNNLogLoss"] == 1.5 and v["RCNNL1LossCRCNN"] == 2.5
    assert math.isnan(v["AutoFocusAcc"]) and math.isnan(v["AutoFocusLogLoss"])
    single = metric.RCNNLogLossMetric(None)
    single.bind(acc)
    assert single.get() == ("RCNNLogLoss", 1.5)
    single.reset()                          # one metric zeroes its own slot only
    assert math.isnan(single.get()[1]) and dict(m.get_name_value())["RPNAcc"] == 0.75
    m.reset()
    assert int(acc.buf.abs().sum()) == 0
    with pytest.raises(RuntimeError, match="not bound"):
        metric.RPNAccMetric().get()


# ---- argument refusals
A = 0x7f0000100000
V = [A + 0x1000 * i for i in range(1, 12)]
ORDER = ("rpn_prob ld_rpn rpn_label B H W A cls_prob ld_cls cls_label N K af_prob ld_af af_label Haf Waf counts "
         "loss_buf acc workspace stream").split()
GOOD = dict(rpn_prob=A, ld_rpn=42, rpn_label=V[0], B=0, H=32, W=32, A=21, cls_prob=V[1], ld_cls=81, cls_label=V[2],
            N=0, K=81, af_prob=V[3], ld_af=2, af_label=V[4], Haf=32, Waf=32, counts=V[5], loss_buf=V[6], acc=V[7],
            workspace=V[8], stream=0)


def _call(**change):
    a = dict(GOOD)
    a.update(change)
    L = _lib.lib()
    rc = L.sniper_train_metric_accum(*[a[k] for k in ORDER])
    return rc, L.sniper_last_error().decode()


def test_empty_step_is_accepted_without_a_launch():
    for change in (dict(), dict(N=5), dict(B=3), dict(af_prob=0, af_label=0, Haf=0, Waf=0, ld_af=0)):
        rc, msg = _call(**change)
        assert rc == 0, (change, msg)


BAD = [
    (dict(B=-1), r"B \(-1\) must not be negative"),
    (dict(N=-1), r"N \(-1\) must not be negative"),
    (dict(H=0), r"H \(0\) and W \(32\) must be positive"),
    (dict(W=-2), r"H \(32\) and W \(-2\) must be positive"),
    (dict(A=0), r"A \(0\) must be at least 1"),
    (dict(K=0), r"K \(0\) must be at least 1"),
    (dict(ld_rpn=41), r"ld of rpn_prob \(41\) is smaller than 2A \(42\)"),
    (dict(ld_cls=80), r"ld of cls_prob \(80\) is smaller than K \(81\)"),
    (dict(rpn_prob=0), r"rpn_prob must not be null"),
    (dict(rpn_label=0), r"rpn_label must not be null"),
    (dict(cls_prob=0), r"cls_prob must not be null"),
    (dict(cls_label=0), r"cls_label must not be null"),
    (dict(counts=0), r"counts must not be null"),
    (dict(loss_buf=0), r"loss_buf must not be null"),
    (dict(acc=0), r"acc must not be null"),
    (dict(workspace=0), r"workspace must not be null"),
    (dict(af_label=0), r"af_label must not be null when af_prob is given"),
    (dict(Haf=0), r"Haf \(0\) and Waf \(32\) must be positive"),
    (dict(ld_af=1), r"ld of af_prob \(1\) is smaller than 2"),
    (dict(B=100000), r"B\*H\*W\*A \(2150400000\) must be below 2\^31"),
    (dict(B=2, Haf=40000, Waf=40000), r"B\*Haf\*Waf \(\d+\) must be below 2\^31"),
]


@pytest.mark.parametrize("change,pattern", BAD, ids=["-".join("%s=%s" % kv for kv in c.items()) for c, _ in BAD])
def test_one_violated_rule_is_refused_by_name(change, pattern):
    for size in (dict(B=0, N=0), dict(B=2, N=600)):     # refused before the empty-step shortcut as well
        args = dict(size)
        args.update(change)
        rc, msg = _call(**args)
        assert rc != 0, args
        assert re.search("train_metric_accum: " + pattern, msg), msg
