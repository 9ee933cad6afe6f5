"""Trainer.fit's loop, Speedometer and module_checkpoint without a device: a fake trainer whose step adds known terms
to a host accumulator, an iterator whose chip count changes between epochs, `.states` files of a real parameter store
(built over the float64 stand-ins of the kernels), and a world-size-2 gloo run."""
import logging
import os
import sys
import time

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from sniper_b200 import callback, checkpoint, iterator, metric, trainer  # noqa: E402


# ---------------------------------------------------------------- Speedometer (MXNet 1.2 callback.py:120-170)
class _Clock(object):
    def __init__(self):
        self.t = 100.0

    def __call__(self):
        return self.t


def _speedometer_lines(monkeypatch, caplog, frequent, epochs):
    clock = _Clock()
    monkeypatch.setattr(callback.time, "time", clock)
    acc = metric.MetricAccumulator("cpu")
    m = metric.CompositeEvalMetric([metric.RPNAccMetric(), metric.RPNL1LossMetric()])
    m.bind(acc)
    sp = callback.Speedometer(4, frequent)
    caplog.set_level(logging.INFO)
    caplog.clear()
    resets = []
    for epoch, n in epochs:
        for nbatch in range(n):
            clock.t += 0.5
            acc.buf[0] += 2
            acc.buf[8] += 1
            acc.buf[2] += 2
            acc.buf[16 + 2:16 + 3].view(torch.float64).add_(1.0)
            before = int(acc.buf[0])
            sp(trainer.BatchEndParam(epoch=epoch, nbatch=nbatch, eval_metric=m, locals=None))
            if before and int(acc.buf[0]) == 0:
                resets.append((epoch, nbatch))
    return [r.getMessage() for r in caplog.records], resets


def test_speedometer_every_batch(monkeypatch, caplog):
    lines, resets = _speedometer_lines(monkeypatch, caplog, 1, [(0, 3)])
    # the first call only starts the clock; then every batch: 1 batch x 4 samples / 0.5 s, the metrics of that batch
    assert lines == ["Epoch[0] Batch [1]\tSpeed: 8.00 samples/sec\tRPNAcc=0.500000\tRPNL1Loss=0.500000",
                     "Epoch[0] Batch [2]\tSpeed: 8.00 samples/sec\tRPNAcc=0.500000\tRPNL1Loss=0.500000"]
    assert resets == [(0, 1), (0, 2)]


def test_speedometer_every_20_and_restart_at_a_new_epoch(monkeypatch, caplog):
    lines, resets = _speedometer_lines(monkeypatch, caplog, 20, [(0, 45), (1, 25)])
    # epoch 0: clock starts at batch 0, prints at 20 (window 1..20) and 40 (21..40); the metrics then hold only the
    # window since the last reset.  Epoch 1: the batch count drops, so the clock restarts at batch 0 and prints at 20.
    # The accumulated metrics are NOT reset by the restart (as in MXNet): batches 41..44 of epoch 0 count in epoch 1's
    # first window.
    assert lines == ["Epoch[0] Batch [20]\tSpeed: 8.00 samples/sec\tRPNAcc=0.500000\tRPNL1Loss=0.500000",
                     "Epoch[0] Batch [40]\tSpeed: 8.00 samples/sec\tRPNAcc=0.500000\tRPNL1Loss=0.500000",
                     "Epoch[1] Batch [20]\tSpeed: 8.00 samples/sec\tRPNAcc=0.500000\tRPNL1Loss=0.500000"]
    assert resets == [(0, 20), (0, 40), (1, 20)]


# ---------------------------------------------------------------- fit on a fake trainer
class _P(object):
    def __init__(self):
        self.total = 12
        self.w = torch.arange(12, dtype=torch.float32) * 0.25
        self.g = torch.zeros(12)
        self.mom = torch.arange(12, dtype=torch.float32) * -0.5


class _Net(object):
    """bbox_pred weight [4, 2] = P[0:8] stored transposed, bias [4] = P[8:12] (a layout conversion to invert)."""

    def __init__(self, autofocus=False):
        self.cfg = type("C", (), {"autofocus": autofocus})()
        self.P = _P()

    def export_reference(self, grads=False):
        src = self.P.g if grads else self.P.w
        arg = {"bbox_pred_weight": src[:8].view(2, 4).t().numpy().copy(), "bbox_pred_bias": src[8:].numpy().copy()}
        return arg, ({} if grads else {"bn_moving_mean": np.ones(3, np.float32)})


class _Done(object):
    def synchronize(self):
        pass


def _fake_trainer(autofocus=False):
    t = trainer.Trainer.__new__(trainer.Trainer)
    t.device, t.world_size, t.metric_acc, t.g_up, t.g_metric = torch.device("cpu"), 1, None, None, None
    t.net, t.num_update, t.steps = _Net(autofocus), 0, []

    def step(raw, input_stage, lr=None):
        t.num_update += 1
        t.steps.append(raw)
        b = t.metric_acc.buf
        b[0:6] += 2                       # two valid rows per step in every problem
        b[8] += raw % 3                   # RPN hits
        b[16 + 1:16 + 2].view(torch.float64).add_(float(raw))
        return _Done()
    t.step_raw_async = step
    return t


class _Chips(object):
    """A resettable iterator whose batch count differs from epoch to epoch (the negative-chip draw)."""

    def __init__(self, counts):
        self.counts, self.epoch, self.i = list(counts), 0, 0

    def __iter__(self):
        return self

    def __next__(self):
        if self.i >= self.counts[self.epoch]:
            raise StopIteration
        self.i += 1
        return 100 * self.epoch + self.i

    def reset(self):
        self.epoch, self.i = self.epoch + 1, 0


@pytest.mark.parametrize("prefetch", [False, True])
def test_fit_follows_epoch_markers_and_writes_epoch_files(tmp_path, caplog, prefetch):
    caplog.set_level(logging.INFO)
    t = _fake_trainer()
    chips = _Chips([5, 3])
    it = iterator.PrefetchingIter(chips, depth=2, epochs=2, epoch_marker=True) if prefetch else chips
    seen = []
    ends = []
    prefix = str(tmp_path / "e2e")
    try:
        t.fit(it, None, 2, eval_metric=None,
              batch_end_callback=lambda p: seen.append((p.epoch, p.nbatch)),
              epoch_end_callback=[lambda e, s, a, x: ends.append(e), callback.module_checkpoint(t, prefix)])
    finally:
        if prefetch:
            it.close()
    assert seen == [(0, i) for i in range(5)] + [(1, i) for i in range(3)]
    assert t.steps == [1, 2, 3, 4, 5, 101, 102, 103] and ends == [0, 1]
    msgs = [r.getMessage() for r in caplog.records]
    # epoch 1 alone: the metrics were reset at the epoch start; RPNLogLoss = (101 + 102 + 103) / 6
    assert "Epoch[1] Train-RPNLogLoss=%f" % (306 / 6.0) in msgs and "Epoch[0] Train-RPNAcc=%f" % (6 / 10.0) in msgs
    assert [m.split("=")[0] for m in msgs if m.startswith("Epoch[0] T")] == [
        "Epoch[0] Train-RPNAcc", "Epoch[0] Train-RPNLogLoss", "Epoch[0] Train-RPNL1Loss", "Epoch[0] Train-RCNNAcc",
        "Epoch[0] Train-RCNNLogLoss", "Epoch[0] Train-RCNNL1LossCRCNN", "Epoch[0] Time cost"]
    arg, aux = checkpoint.load_param(prefix, 1)
    assert {"bbox_pred_weight_test", "bbox_pred_bias_test"} <= set(arg) and "bn_moving_mean" in aux
    assert os.path.exists(prefix + "-0001.states") and os.path.exists(prefix + "-0002.states")
    t2 = _fake_trainer()
    t2.load_optimizer_states(prefix + "-0001.states")
    assert t2.num_update == 5


def test_fit_refuses_a_prefetcher_without_markers():
    chips = _Chips([2])
    it = iterator.PrefetchingIter(chips, depth=1, epochs=1)
    try:
        with pytest.raises(ValueError, match="epoch_marker"):
            _fake_trainer().fit(it, None, 1)
    finally:
        it.close()


def test_fit_refuses_a_raw_batch_ring_too_small_for_two_steps_in_flight():
    """fit has two steps in flight, each reading its raw batch through asynchronous H2D copies: behind a prefetcher of
    depth d the iterator needs d + 3 raw buffers, or a buffer could be refilled while its copy is still running."""
    for n, ok in ((4, False), (5, True)):
        chips = _Chips([2])
        chips._buffers = [None] * n
        it = iterator.PrefetchingIter(chips, depth=2, epochs=1, epoch_marker=True)
        try:
            if ok:
                _fake_trainer().fit(it, None, 1)
            else:
                with pytest.raises(ValueError, match="owns 4 raw buffers; with prefetch depth 2 it needs 5"):
                    _fake_trainer().fit(it, None, 1)
        finally:
            it.close()


def test_states_round_trip_on_a_real_parameter_store(tmp_path, monkeypatch):
    """Momenta through export_reference's own conversions (MobileNetV2: padded rows, depthwise and head layouts) and
    back, byte-equal; num_update as int64; the gradient buffer is left as it was."""
    import fake_ops
    from sniper_b200 import model_mnv2, ops
    fake_ops.install(monkeypatch, ops)
    cfg = model_mnv2.MCfg()
    cfg.batch_images = 1
    net = model_mnv2.SniperMobileNetV2(cfg, device="cpu", seed=1)
    P = net.P
    index = checkpoint._momentum_index(net)
    live = np.zeros(P.total, bool)
    for v in index.values():
        live[v.reshape(-1)] = True
    rng = np.random.RandomState(0)
    mom = np.where(live, rng.normal(size=P.total), 0).astype(np.float32)
    P.mom.copy_(torch.from_numpy(mom))
    P.g.copy_(torch.from_numpy(rng.normal(size=P.total).astype(np.float32)))
    g0 = P.g.clone()
    path = str(tmp_path / "x-0003.states")
    checkpoint.save_optimizer_states(path, net, 1234)
    names = [k for k, _ in checkpoint.read_list(path)]
    assert names[-1] == "num_update" and all(k.startswith("mom:") for k in names[:-1])
    assert set(k[4:] for k in names[:-1]) == set(net.export_reference(grads=True)[0])
    P.mom.zero_()
    assert checkpoint.load_optimizer_states(path, net) == 1234
    assert P.mom.numpy().tobytes() == mom.tobytes() and torch.equal(P.g, g0)


# ---------------------------------------------------------------- two ranks
def _rank(rank, world, port, out_dir, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_fit_cpu as F
    t = F._fake_trainer()
    t.world_size = world
    chips = F._Chips([4])
    lines = []
    h = logging.Handler()
    h.emit = lambda r: lines.append(r.getMessage())
    logging.getLogger().addHandler(h)
    logging.getLogger().setLevel(logging.INFO)
    vals = []
    t.fit(chips, None, 1, batch_end_callback=[callback.Speedometer(2, 2),
                                               lambda p: vals.append(dict(p.eval_metric.get_name_value()))],
          epoch_end_callback=callback.module_checkpoint(t, os.path.join(out_dir, "r")))
    q.put((rank, vals[-1]["RPNLogLoss"], vals[-1]["RPNAcc"], len(lines)))
    dist.destroy_process_group()


def test_two_ranks_sum_the_metrics_and_only_rank0_writes(tmp_path):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank, args=(r, 2, 29641, str(tmp_path), q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in procs)
    for p in procs:
        p.join(60)
    # both ranks ran raws 1..4; the Speedometer reset the metrics after batch 2 (raw 3), so the last read covers raw 4
    # of both ranks: log-loss 4 * 2 / (2 * 2), accuracy (4 % 3) * 2 / (2 * 2)
    assert [r[0] for r in res] == [0, 1]
    assert all(r[1] == 2.0 and r[2] == 0.5 for r in res), res
    assert res[0][3] > 0 and res[1][3] == 0          # only rank 0 logs
    assert sorted(os.listdir(str(tmp_path))) == ["r-0001.params", "r-0001.states"]
