"""The reference's training metrics (lib/train_utils/metric.py) as views onto one device accumulator.

`sniper_train_metric_accum` (csrc/train_metric.cu) adds every step's terms into an int64 / float64 accumulator that the
trainer owns; the classes below keep MXNet 1.2's `EvalMetric` surface (SNIPER-mxnet/python/mxnet/metric.py:68-180,
CompositeEvalMetric :230-345) but their `update` does nothing -- the trainer's launch already did the work, without a
host copy per step.  `get()` makes one non-blocking D2H copy of the accumulator into pinned memory and waits for that
copy only; with several ranks it first sums the accumulator over them (what executor_group's `update_metric` does by
updating one metric from every device).  `reset()` zeroes the metric's slots on the stream.
"""
import numpy as np
import torch

# slot of each metric in the accumulator (csrc/train_metric.cu)
SLOTS = {"RPNAcc": 0, "RPNLogLoss": 1, "RPNL1Loss": 2, "RCNNAcc": 3, "RCNNLogLoss": 4, "RCNNL1LossCRCNN": 5,
         "AutoFocusAcc": 6, "AutoFocusLogLoss": 7}
_HIT_SLOTS = (0, 3, 6)        # accuracies: sum_metric is the int64 hit count


class MetricAccumulator(object):
    """int64 num_inst[8] | int64 hits[8] | float64 sum[8] on `device`, plus the kernel's scratch."""

    def __init__(self, device, world_size=1):
        from . import ops
        self.device = torch.device(device)
        self.world_size = world_size
        self.buf = torch.zeros(24, dtype=torch.int64, device=self.device)
        self.workspace = ops.train_metric_workspace(self.device) if self.device.type == "cuda" else None
        self.host = torch.zeros(24, dtype=torch.int64)
        if self.device.type == "cuda":
            self.host = self.host.pin_memory()

    def reset(self, slots=None):
        if slots is None:
            self.buf.zero_()
        else:
            self.buf.view(3, 8)[:, list(slots)] = 0

    def read(self):
        """-> (num_inst int64 [8], sum_metric float64 [8]) summed over the ranks."""
        buf = self.buf
        if self.world_size > 1:
            buf = buf.clone()
            torch.distributed.all_reduce(buf[:16])
            torch.distributed.all_reduce(buf[16:].view(torch.float64))
        if self.device.type == "cuda":
            self.host.copy_(buf, non_blocking=True)
            done = torch.cuda.Event()
            done.record()
            done.synchronize()
        else:
            self.host.copy_(buf)
        h = self.host.numpy().copy()
        sums = h[16:].view(np.float64).copy()
        sums[list(_HIT_SLOTS)] = h[8:16][list(_HIT_SLOTS)]
        return h[:8], sums


def _value(num, sums, slot):
    return float("nan") if num[slot] == 0 else float(sums[slot] / num[slot])


class EvalMetric(object):
    """mxnet.metric.EvalMetric over one accumulator slot (bound by `Trainer.fit`)."""

    def __init__(self, name):
        self.name = name
        self.slot = SLOTS[name]
        self.acc = None

    def bind(self, acc):
        self.acc = acc

    def _bound(self):
        if self.acc is None:
            raise RuntimeError("%s is not bound to a trainer's accumulator (Trainer.fit binds it)" % self.name)
        return self.acc

    def update(self, labels, preds):
        """No-op: the trainer's per-step launch accumulates on the device."""

    def reset(self):
        if self.acc is not None:
            self.acc.reset([self.slot])

    def _get(self, num, sums):
        return self.name, _value(num, sums, self.slot)

    def get(self):
        return self._get(*self._bound().read())

    def get_name_value(self):
        name, value = self.get()
        if not isinstance(name, list):
            name = [name]
        if not isinstance(value, list):
            value = [value]
        return list(zip(name, value))

    def __str__(self):
        return "EvalMetric: {}".format(dict(self.get_name_value()))


class RPNAccMetric(EvalMetric):
    def __init__(self):
        super(RPNAccMetric, self).__init__("RPNAcc")


class RPNLogLossMetric(EvalMetric):
    def __init__(self):
        super(RPNLogLossMetric, self).__init__("RPNLogLoss")


class RPNL1LossMetric(EvalMetric):
    def __init__(self):
        super(RPNL1LossMetric, self).__init__("RPNL1Loss")


class RCNNAccMetric(EvalMetric):
    def __init__(self, cfg=None):
        super(RCNNAccMetric, self).__init__("RCNNAcc")


class RCNNLogLossMetric(EvalMetric):
    def __init__(self, cfg=None):
        super(RCNNLogLossMetric, self).__init__("RCNNLogLoss")


class RCNNL1LossCRCNNMetric(EvalMetric):
    def __init__(self, cfg=None):
        super(RCNNL1LossCRCNNMetric, self).__init__("RCNNL1LossCRCNN")


class AutoFocusAccMetric(EvalMetric):
    def __init__(self):
        super(AutoFocusAccMetric, self).__init__("AutoFocusAcc")


class AutoFocusLogLossMetric(EvalMetric):
    def __init__(self):
        super(AutoFocusLogLossMetric, self).__init__("AutoFocusLogLoss")


class CompositeEvalMetric(EvalMetric):
    """mxnet.metric.CompositeEvalMetric: one accumulator read serves every child."""

    def __init__(self, metrics=None, name="composite"):
        self.name = name
        self.metrics = list(metrics or [])
        self.acc = None

    def add(self, metric):
        self.metrics.append(metric)
        if self.acc is not None:
            metric.bind(self.acc)

    def get_metric(self, index):
        return self.metrics[index]

    def bind(self, acc):
        self.acc = acc
        for m in self.metrics:
            m.bind(acc)

    def reset(self):
        if self.acc is not None:
            self.acc.reset([m.slot for m in self.metrics])

    def get(self):
        num, sums = self._bound().read()
        names, values = [], []
        for m in self.metrics:
            name, value = m._get(num, sums)
            names.append(name)
            values.append(value)
        return names, values


def default_metrics(autofocus=False):
    """The composite main_train.py builds (:104-128) for an end-to-end run (not TRAIN.ONLY_PROPOSAL, no mask)."""
    m = CompositeEvalMetric()
    for x in (RPNAccMetric(), RPNLogLossMetric(), RPNL1LossMetric(), RCNNAccMetric(), RCNNLogLossMetric(),
              RCNNL1LossCRCNNMetric()):
        m.add(x)
    if autofocus:
        m.add(AutoFocusAccMetric())
        m.add(AutoFocusLogLossMetric())
    return m
