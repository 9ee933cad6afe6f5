"""sniper_train_metric_accum on the device: against the reference classes' fixture and the float64 restatement at the
real step shapes (ResNet-101 B = 20, MobileNetV2 B = 40, the AutoFocus map), run-to-run bytes, graph replays, reset,
and the AutoFocus hit count against sniper_focus_acc."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import train_metric_np as T  # noqa: E402
from sniper_b200 import metric, ops  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOGLOSS = [1, 4, 7]


def _run(c, acc=None, times=1):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    A = c["A"]
    counts = [int((np.asarray(c["rpn_label"]) != -1).sum()), int((np.asarray(c["cls_label"]) != -1).sum())]
    if c.get("af_prob") is not None:
        counts.append(int((np.asarray(c["af_label"]) != -1).sum()))
    loss = torch.zeros(8, device=DEV)
    loss[1], loss[3] = float(np.float32(c["rpn_l1"])), float(np.float32(c["rcnn_l1"]))
    acc = acc or metric.MetricAccumulator(DEV)
    args = [t(c["rpn_prob"]), t(c["rpn_label"]), A, t(c["cls_prob"]), t(c["cls_label"]),
            torch.tensor(counts, dtype=torch.int32, device=DEV), loss, acc.buf, acc.workspace]
    kw = dict(af_prob=None if c.get("af_prob") is None else t(c["af_prob"]),
              af_label=None if c.get("af_label") is None else t(c["af_label"]))
    for _ in range(times):
        ops.train_metric_accum(*args, **kw)
    torch.cuda.synchronize()
    return acc, args, kw


def _host(acc):
    h = acc.buf.cpu().numpy()
    return h[:8], h[8:16], h[16:].view(np.float64)


def _check(c, acc):
    num, hits, sums = _host(acc)
    enum, es = T.step(**c)
    assert np.array_equal(num, enum)
    assert np.array_equal(hits[[0, 3, 6]], es[[0, 3, 6]].astype(np.int64))
    for k in LOGLOSS:
        assert abs(sums[k] - es[k]) <= 1e-12 * abs(es[k]), (k, sums[k], es[k])
    assert sums[2] == es[2] and sums[5] == es[5]


def _fixture_case(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", "train_metric_ref.npz"))
    g = lambda k: z[name + "/" + k]
    af = (name + "/af_prob") in z
    c = dict(rpn_prob=g("rpn_prob"), rpn_label=g("rpn_label"), A=int(g("A")), cls_prob=g("cls_prob"),
             cls_label=g("cls_label"), rpn_l1=g("rpn_l1"), rcnn_l1=g("rcnn_l1"),
             af_prob=g("af_prob") if af else None, af_label=g("af_label") if af else None)
    return c, g("sum_metric"), g("num_inst")


@pytest.mark.parametrize("name", ["resnet101_af", "mobilenetv2", "ignored"])
def test_kernel_against_the_reference_fixture(name):
    c, ref_sum, ref_num = _fixture_case(name)
    acc, _, _ = _run(c)
    num, hits, sums = _host(acc)
    n = 8 if c["af_prob"] is not None else 6
    assert np.array_equal(num[:n], ref_num[:n])
    for k in ((0, 3, 6) if n == 8 else (0, 3)):
        assert hits[k] == ref_sum[k]
    _check(c, acc)


def _synthetic(B, H, A, N, K, af, seed):
    rng = np.random.RandomState(seed)

    def two(Bq, Hq, Aq):
        p = rng.dirichlet([1, 1], size=(Bq, Hq, Hq, Aq)).astype(np.float32)
        flat = p.reshape(-1, 2)
        flat[rng.rand(flat.shape[0]) < 0.03] = (0.5, 0.5)
        flat[rng.rand(flat.shape[0]) < 0.03] = (0.0, 1.0)
        prob = np.ascontiguousarray(p.transpose(0, 1, 2, 4, 3).reshape(Bq, Hq, Hq, 2 * Aq))
        return prob, rng.choice([-1, -1, -1, 0, 1], size=(Bq, Aq * Hq * Hq)).astype(np.float32)
    prob, lab = two(B, H, A)
    cls = rng.dirichlet(np.ones(K), size=N).astype(np.float32)
    cls[: N // 20, :] = 1.0 / K
    clab = rng.randint(-1, K, N).astype(np.float32)
    c = dict(rpn_prob=prob, rpn_label=lab, A=A, cls_prob=cls, cls_label=clab, rpn_l1=np.float32(12.5),
             rcnn_l1=np.float32(3.25), af_prob=None, af_label=None)
    if af:
        c["af_prob"], c["af_label"] = two(B, H, 1)
    return c


SHAPES = {"resnet101_b20": (20, 32, 21, 6000, 81, False), "resnet101_b20_autofocus": (20, 32, 21, 6000, 81, True),
          "mobilenetv2_b40": (40, 16, 15, 12000, 81, False)}


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_real_shapes_against_the_restatement_and_run_to_run(name):
    c = _synthetic(*SHAPES[name], seed=len(name))
    a1, _, _ = _run(c)
    _check(c, a1)
    a2, _, _ = _run(c)
    assert a1.buf.cpu().numpy().tobytes() == a2.buf.cpu().numpy().tobytes()


def test_graph_replays_add_exact_multiples_and_reset_zeroes():
    c = _synthetic(*SHAPES["resnet101_b20_autofocus"], seed=7)
    one, args, kw = _run(c)
    acc = metric.MetricAccumulator(DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            ops.train_metric_accum(*(args[:7] + [acc.buf, acc.workspace]), **kw)
    torch.cuda.synchronize()
    acc.reset()
    for _ in range(5):
        g.replay()
    torch.cuda.synchronize()
    n1, h1, _ = _host(one)
    n5, h5, s5 = _host(acc)
    assert np.array_equal(n5, 5 * n1) and np.array_equal(h5, 5 * h1)
    e = T.step(**c)[1]
    assert abs(s5[1] - 5 * e[1]) <= 1e-12 * 5 * e[1]
    m = metric.default_metrics(True)
    m.bind(acc)
    m.reset()
    torch.cuda.synchronize()
    assert int(acc.buf.abs().sum()) == 0


def test_autofocus_hits_equal_focus_acc():
    c = _synthetic(*SHAPES["resnet101_b20_autofocus"], seed=9)
    acc, _, kw = _run(c)
    counts = torch.zeros(2, device=DEV)
    ops.focus_acc(kw["af_prob"], kw["af_label"], counts)
    torch.cuda.synchronize()
    num, hits, _ = _host(acc)
    assert hits[6] == int(counts[0].item()) and num[6] == int(counts[1].item())
