"""Runs the reference's own lib/train_utils/metric.py, unchanged, on seeded step outputs and writes
tests/golden/train_metric_ref.npz.

The reference module needs `mxnet` for three things only; a minimal stub provides them:
  * `mx.metric.EvalMetric`, restated from SNIPER-mxnet/python/mxnet/metric.py:68-180 (name, sum_metric, num_inst,
    reset, get with NaN on zero instances, get_name_value);
  * `mx.ndarray.argmax_channel` (argmax over axis 1, first maximum on ties);
  * `.asnumpy()` / `.shape` of the arrays handed to `update` (plain numpy underneath).

The inputs are laid out as the reference's executor hands them to `update_metric`: rpn_cls_prob [B, 2, A*H, W],
scale_cls_prob [B, 2, H, W], rcnn_cls_prob [N, K], labels [B, A*H*W] / [B, H*W] / [N].  The fixture stores them in this
package's layouts (NHWC probabilities) next to each metric's sum_metric and num_inst.

usage: python oracle/run_ref_metric.py [/path/to/reference]
"""
import importlib.util
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("RPNAcc", "RPNLogLoss", "RPNL1Loss", "RCNNAcc", "RCNNLogLoss", "RCNNL1LossCRCNN", "AutoFocusAcc",
         "AutoFocusLogLoss")


class _ND(object):
    def __init__(self, a):
        self.a = np.asarray(a)
        self.shape = self.a.shape

    def asnumpy(self):
        return self.a.copy()


class EvalMetric(object):
    def __init__(self, name, output_names=None, label_names=None, **kwargs):
        self.name = str(name)
        self.reset()

    def reset(self):
        self.num_inst = 0
        self.sum_metric = 0.0

    def get(self):
        if self.num_inst == 0:
            return (self.name, float('nan'))
        return (self.name, self.sum_metric / self.num_inst)

    def get_name_value(self):
        name, value = self.get()
        return list(zip([name], [value]))


def _stub():
    mx = types.ModuleType("mxnet")
    mx.metric = types.SimpleNamespace(EvalMetric=EvalMetric)
    mx.ndarray = types.SimpleNamespace(argmax_channel=lambda x: _ND(np.argmax(x.a, axis=1).astype(np.float32)))
    mx.nd = mx.ndarray
    return mx


def _load(ref):
    sys.modules["mxnet"] = _stub()
    spec = importlib.util.spec_from_file_location("ref_metric", os.path.join(ref, "lib", "train_utils", "metric.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _softmax(z):
    e = np.exp(z - z.max(-1, keepdims=True))
    return (e / e.sum(-1, keepdims=True)).astype(np.float32)


def _two_way(rng, B, H, W, A, ignore_all):
    """NHWC prob [B,H,W,2A] (bg channel a, fg A+a) with exact ties and p = 0 entries, labels [B, A*H*W]."""
    p = _softmax(rng.normal(0, 2, (B, H, W, A, 2)))
    flat = p.reshape(-1, 2)
    n = flat.shape[0]
    flat[rng.choice(n, n // 20, replace=False)] = (0.5, 0.5)
    flat[rng.choice(n, n // 20, replace=False)] = (0.0, 1.0)
    flat[rng.choice(n, n // 20, replace=False)] = (1.0, 0.0)
    prob = np.ascontiguousarray(p.transpose(0, 1, 2, 4, 3).reshape(B, H, W, 2 * A))
    lab = rng.choice([-1, -1, 0, 1], size=(B, A * H * W)).astype(np.float32)
    if ignore_all:
        lab[:] = -1
    return prob, lab


def _rcnn(rng, N, K, ignore_all):
    z = rng.normal(0, 2, (N, K))
    z[: N // 10, 3] = z[: N // 10, 7] = z[: N // 10].max(1) + 1.0        # equal maxima
    p = _softmax(z)
    p[N // 10: N // 5, :] = 1.0 / K                                         # every class tied
    rows = np.arange(N // 5, N // 4)
    lab = rng.randint(-1, K, N).astype(np.float32)
    p[rows, lab[rows].astype(int).clip(0)] = 0.0                          # p[label] = 0: the 1e-14 floor
    if ignore_all:
        lab[:] = -1
    return p, lab


def _reference_layout(prob, A):
    """NHWC [B,H,W,2A] -> the reference's rpn_cls_prob [B, 2, A*H, W]."""
    B, H, W = prob.shape[:3]
    return np.ascontiguousarray(prob.reshape(B, H, W, 2, A).transpose(0, 3, 4, 1, 2).reshape(B, 2, A * H, W))


CASES = (  # name, seed, B, H, A, N, K, autofocus, ignore_all
    ("resnet101_af", 1, 1, 32, 21, 300, 81, True, False),
    ("mobilenetv2", 2, 2, 16, 15, 600, 81, False, False),
    ("ignored", 3, 1, 32, 21, 300, 81, True, True),
)


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    M = _load(ref)
    out = {}
    for name, seed, B, H, A, N, K, af, ign in CASES:
        rng = np.random.RandomState(seed)
        prob, lab = _two_way(rng, B, H, H, A, ign)
        cls, clab = _rcnn(rng, N, K, ign)
        rpn_l1 = rng.uniform(0, 1, (B, 4 * A, H, H)).astype(np.float32)
        rcnn_l1 = rng.uniform(0, 1, (N, 4)).astype(np.float32)
        cfg = types.SimpleNamespace(TRAIN=types.SimpleNamespace(END2END=True, ENABLE_OHEM=False, AUTO_FOCUS=af,
                                                                WITH_MASK=False))
        preds = [_ND(_reference_layout(prob, A)), _ND(rpn_l1)]
        labels = [_ND(lab), None, None, None]
        if af:
            afp, afl = _two_way(rng, B, H, H, 1, ign)
            preds.append(_ND(_reference_layout(afp, 1)))
            labels.append(_ND(afl))
            out[name + "/af_prob"], out[name + "/af_label"] = afp, afl
        preds += [_ND(cls), _ND(rcnn_l1), _ND(clab)]
        metrics = [M.RPNAccMetric(), M.RPNLogLossMetric(), M.RPNL1LossMetric(), M.RCNNAccMetric(cfg),
                   M.RCNNLogLossMetric(cfg), M.RCNNL1LossCRCNNMetric(cfg)]
        if af:
            metrics += [M.AutoFocusAccMetric(), M.AutoFocusLogLossMetric()]
        sums, nums = np.full(8, np.nan), np.zeros(8, np.int64)
        for m in metrics:
            assert m.name in NAMES
            m.update(labels, preds)
            sums[NAMES.index(m.name)] = float(m.sum_metric)
            nums[NAMES.index(m.name)] = int(m.num_inst)
        out.update({name + "/rpn_prob": prob, name + "/rpn_label": lab, name + "/cls_prob": cls,
                    name + "/cls_label": clab, name + "/rpn_l1": np.float32(rpn_l1.sum()),
                    name + "/rcnn_l1": np.float32(rcnn_l1.sum()), name + "/sum_metric": sums, name + "/num_inst": nums,
                    name + "/A": np.int64(A)})
    path = os.path.join(ROOT, "tests", "golden", "train_metric_ref.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
