"""MobileNetV2 training (BASELINE config 4) reproduces itself and resumes byte for byte, in bf16 and in fp32.

* Two runs of a few Trainer steps (CUDA graphs, training metrics on), each in a fresh process, dump byte-identical
  state: weights, bf16 weight copies, gradients, momenta, BatchNorm moving statistics, the last step's rois and labels,
  and the metric accumulator.  The accumulator's two L1 slots are left out: they fold in the smooth-L1 loss sums, which
  are fp32-atomic scalars with last-bit run-to-run noise (DESIGN "Reproducibility"); nothing the step computes reads
  them.
* fit-style resume, as tests/test_fit_gpu.py does for ResNet-101: N + M continuous steps; N steps, a checkpoint (.params
  + .states); a fresh net with different initial weights loads both and takes M more steps.  Weights, momenta, moving
  statistics, lr, num_update and the bf16 copies must equal the continuous run's bytes.
Every case runs in its own process, so no earlier net in the process can affect it."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
L1_SUM_SLOTS = (16 + 2, 16 + 5)      # metric.MetricAccumulator.buf: num_inst[8] | hits[8] | sum[8]; RPNL1Loss, RCNNL1Loss


def _run(code, tmp_path):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.dirname(os.path.abspath(__file__))]))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def _net(bf16, seed, B=2):
    from sniper_b200 import model_mnv2
    c = model_mnv2.MCfg()
    c.batch_images, c.bf16 = B, bool(bf16)
    return model_mnv2.SniperMobileNetV2(c, device=DEV, seed=seed)


def _batches(net, n, B=2):
    from sniper_b200 import synth_batch
    return [synth_batch.make_batch(B, seed=40 + i, device="cpu", pinned=True, A=net.cfg.num_anchors,
                                   stride=net.cfg.feat_stride) for i in range(n)]


def _dump_case(bf16, path, steps=4):
    """Run `steps` graph-replayed steps with metrics and write every tensor of the state to `path` (.npz)."""
    import torch
    from sniper_b200 import trainer
    net = _net(bf16, 3)
    batches = _batches(net, steps)
    tr = trainer.Trainer(net.cfg, device=DEV, net=net, scheduler=lambda n: 0.001 * (1 + (n >= 2)), metrics=True)
    for i, b in enumerate(batches):
        tr.step(b, prefetch=batches[i + 1] if i + 1 < len(batches) else None)
    torch.cuda.synchronize()
    assert tr.g_fb is not None, "the steps did not run as CUDA graphs"
    arg, aux = net.export_reference()
    h = lambda t: t.detach().cpu().numpy()
    acc = h(tr.metric_acc.buf).copy()
    acc[list(L1_SUM_SLOTS)] = 0
    state = dict(w=h(net.P.w), g=h(net.P.g), mom=h(net.P.mom), rois=h(tr.out["rois"]), label=h(tr.out["label"]),
                 metric=acc, num_update=np.int64(tr.num_update))
    if net.P.w16 is not None:
        state["w16"] = h(net.P.w16.float())
    for k in sorted(aux):
        state["aux:" + k] = np.asarray(aux[k])
    np.savez(path, **state)


@pytest.mark.parametrize("bf16", [True, False], ids=["bf16", "fp32"])
def test_two_fresh_processes_give_identical_state(bf16, tmp_path):
    paths = [str(tmp_path / ("run%d.npz" % i)) for i in range(2)]
    for p in paths:
        _run("import test_mnv2_reproducible_gpu as R; R._dump_case(%r, %r)" % (bf16, p), tmp_path)
    a, b = np.load(paths[0]), np.load(paths[1])
    assert sorted(a.files) == sorted(b.files)
    differ = [k for k in a.files if a[k].tobytes() != b[k].tobytes()]
    assert differ == [], differ
    assert a["num_update"] == 4 and np.isfinite(a["w"]).all() and a["g"].any()


def _state(tr):
    net = tr.net
    _, aux = net.export_reference()
    return dict(weights=net.P.w.cpu().numpy().tobytes(), momenta=net.P.mom.cpu().numpy().tobytes(),
                moving=b"".join(np.asarray(aux[k]).tobytes() for k in sorted(aux)), lr=np.float64(tr.lr).tobytes(),
                num_update=tr.num_update,
                w16=None if net.P.w16 is None else net.P.w16.float().cpu().numpy().tobytes())


def _resume_case(bf16, tmp_path):
    import torch
    from sniper_b200 import callback, checkpoint, trainer
    N, M = 2, 2
    net0 = _net(bf16, 3)
    batches = _batches(net0, N + M)
    sched = lambda n: 0.001 * (1 + (n >= 3))             # the lr changes between the two halves
    tr = trainer.Trainer(net0.cfg, device=DEV, net=net0, scheduler=sched)
    for b in batches:
        tr.step(b)
    torch.cuda.synchronize()
    ref = _state(tr)
    del tr, net0

    net1 = _net(bf16, 3)
    tr1 = trainer.Trainer(net1.cfg, device=DEV, net=net1, scheduler=sched)
    for b in batches[:N]:
        tr1.step(b)
    prefix = os.path.join(tmp_path, "r")
    callback.module_checkpoint(tr1, prefix)(N - 1)
    del tr1, net1

    net2 = _net(bf16, 11)                                  # different initial weights: everything must come from disk
    arg, aux = checkpoint.load_param(prefix, N)
    net2.load_reference(arg, aux)
    tr2 = trainer.Trainer(net2.cfg, device=DEV, net=net2, scheduler=sched)
    tr2.load_optimizer_states("%s-%04d.states" % (prefix, N))
    for b in batches[N:]:
        tr2.step(b)
    torch.cuda.synchronize()
    got = _state(tr2)
    for k in ref:
        assert ref[k] == got[k], k


@pytest.mark.parametrize("bf16", [True, False], ids=["bf16", "fp32"])
def test_resumed_run_continues_byte_equal(bf16, tmp_path):
    _run("import test_mnv2_reproducible_gpu as R; R._resume_case(%r, %r)" % (bf16, str(tmp_path)), tmp_path)
