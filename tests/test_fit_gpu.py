"""Trainer.fit and resume on the device: N + M continuous steps equal N steps, a checkpoint (.params + .states), a fresh
net loading both and M more steps, byte for byte; two short epochs of fit from the iterator (ResNet-101 with and
without AutoFocus, MobileNetV2) with every Speedometer window checked against the float64 restatement."""
import logging
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import train_metric_np as T  # noqa: E402
from sniper_b200 import callback, checkpoint, metric, model, model_mnv2, synth_batch, trainer  # noqa: E402
from sniper_b200 import iterator as IT  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _net(kind, seed):
    if kind == "mobilenetv2_bf16":
        c = model_mnv2.MCfg()
        c.batch_images, c.bf16 = 2, True
        return model_mnv2.SniperMobileNetV2(c, device=DEV, seed=seed)
    c = model.Cfg()
    c.batch_images, c.bf16 = 2, kind == "resnet101_bf16"
    return model.SniperResNet101(c, device=DEV, seed=seed)


def _state(tr):
    net = tr.net
    arg, aux = net.export_reference()
    return (net.P.w.cpu().numpy().tobytes(), net.P.mom.cpu().numpy().tobytes(),
            b"".join(aux[k].tobytes() for k in sorted(aux)), np.float64(tr.lr).tobytes(), tr.num_update,
            None if net.P.w16 is None else net.P.w16.float().cpu().numpy().tobytes())


def _saved(tr):
    """What a checkpoint must carry, in the reference's names: weights, BatchNorm statistics, momenta, num_update."""
    arg, aux = tr.net.export_reference()
    mom = tr.net.P.mom.cpu().numpy()
    moms = {k: mom[v] for k, v in checkpoint._momentum_index(tr.net).items()}
    return {"arg:" + k: v for k, v in arg.items()}, {"aux:" + k: v for k, v in aux.items()}, moms, tr.num_update


def _diffs(a, b):
    return [k for k in a if a[k].tobytes() != b[k].tobytes()]


# ResNet-101 steps are reproducible run to run (DESIGN "Reproducibility"), so resuming must give the continuous run's
# bytes.  The MobileNetV2 step is not: sniper_depthwise3x3_wgrad sums its per-block partials with fp32 atomics, so two
# continuous runs already differ in the last bits of the depthwise weights, and a near-tied proposal can turn that into
# a different roi and a larger difference later.  For it the checkpoint round trip is checked byte for byte (everything
# the next step reads comes back exactly), and the resumed steps for the schedule and finite weights.
# Each case runs in a fresh process: in a process where TF32 ResNet-101 nets ran before, a bf16 ResNet-101 run no
# longer reproduces itself (DESIGN "Reproducibility"), which would hide what this test checks.
@pytest.mark.parametrize("kind", ["resnet101_tf32", "resnet101_bf16", "mobilenetv2_bf16"])
def test_resume_is_exact(kind, tmp_path):
    import subprocess
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.dirname(os.path.abspath(__file__))]))
    r = subprocess.run([sys.executable, "-c", "import test_fit_gpu as F; F._resume_case(%r, %r)" % (kind, str(tmp_path))],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def _resume_case(kind, tmp_path):
    N, M = 2, 2
    net0 = _net(kind, 3)
    A, stride = net0.cfg.num_anchors, net0.cfg.feat_stride
    batches = [synth_batch.make_batch(2, seed=40 + i, device="cpu", pinned=True, A=A, stride=stride)
               for i in range(N + M)]
    sched = lambda n: 0.001 * (1 + (n >= 3))             # the lr changes between the two halves
    tr = trainer.Trainer(net0.cfg, device=DEV, net=net0, scheduler=sched)
    for b in batches:
        tr.step(b)
    torch.cuda.synchronize()
    ref = _state(tr)
    del tr, net0

    net1 = _net(kind, 3)
    tr1 = trainer.Trainer(net1.cfg, device=DEV, net=net1, scheduler=sched)
    for b in batches[:N]:
        tr1.step(b)
    prefix = os.path.join(tmp_path, "r")
    callback.module_checkpoint(tr1, prefix)(N - 1)
    at_save = _saved(tr1)
    del tr1, net1

    net2 = _net(kind, 11)                                  # different initial weights: everything must come from disk
    arg, aux = checkpoint.load_param(prefix, N)
    net2.load_reference(arg, aux)
    tr2 = trainer.Trainer(net2.cfg, device=DEV, net=net2, scheduler=sched)
    tr2.load_optimizer_states("%s-%04d.states" % (prefix, N))
    at_load = _saved(tr2)
    for a, b in zip(at_save[:3], at_load[:3]):
        assert _diffs(a, b) == []
    assert at_save[3] == at_load[3] == N
    for b in batches[N:]:
        tr2.step(b)
    torch.cuda.synchronize()
    got = _state(tr2)
    names = ("weights", "momenta", "bn moving statistics", "lr", "num_update", "bf16 copies")
    if kind.startswith("resnet101"):
        for name, a, b in zip(names, ref, got):
            assert a == b, (name, _where(net2.P, a, b) if name in ("weights", "momenta") else None)
        return
    assert ref[3:5] == got[3:5]
    assert torch.isfinite(net2.P.w).all() and torch.equal(net2.P.w16, net2.P.w.to(torch.bfloat16))


def _where(P, a, b):
    d = np.nonzero(np.frombuffer(a, np.int32) != np.frombuffer(b, np.int32))[0]
    out = {}
    for name, (o, shape) in P.layout.items():
        k = int(((d >= o) & (d < o + int(np.prod(shape)))).sum())
        if k:
            out[name] = k
    return len(d), sorted(out.items(), key=lambda kv: -kv[1])[:8]


class _Window(object):
    """Before the Speedometer prints: its values must equal the restatement over the steps since the last reset."""

    def __init__(self, tr, sp):
        self.tr, self.sp = tr, sp
        self.num, self.sum = np.zeros(8, np.int64), np.zeros(8)
        self.checked = 0

    def __call__(self, p):
        if p.nbatch == 0:                    # fit reset the metrics at the epoch start
            self.num[:], self.sum[:] = 0, 0
        tr, out = self.tr, self.tr.out
        torch.cuda.synchronize()
        net = tr.net
        h = lambda t: t.detach().cpu().numpy()
        af = out.get("cls_scale_prob")
        n, s = T.step(h(out["rpn_cls_prob"]), h(tr.static["label"]), net.cfg.num_anchors, h(out["cls_prob"]),
                      h(out["label"]), h(net.loss_buf)[1], h(net.loss_buf)[3], None if af is None else h(af),
                      None if af is None else h(out["scale_label"]))
        self.num += n
        self.sum += s
        # the Speedometer's own test (it restarts its clock when the batch count drops)
        if self.sp.init and p.nbatch % self.sp.frequent == 0 and self.sp.last_count <= p.nbatch:
            got = dict(p.eval_metric.get_name_value())
            for name, slot in metric.SLOTS.items():
                if name not in got:
                    continue
                want = float("nan") if self.num[slot] == 0 else self.sum[slot] / self.num[slot]
                assert np.isclose(got[name], want, rtol=1e-12, atol=0, equal_nan=True), (name, got[name], want)
            self.checked += 1
            self.num[:], self.sum[:] = 0, 0


@pytest.mark.parametrize("kind", ["resnet101", "resnet101_autofocus", "mobilenetv2"])
def test_fit_two_epochs_from_the_iterator(kind, tmp_path, caplog):
    caplog.set_level(logging.INFO)
    np.random.seed(5)
    af = kind == "resnet101_autofocus"
    cfg = IT.default_config(autofocus=af, network="mobilenetv2" if kind == "mobilenetv2" else "resnet101")
    B = 2
    roidb = IT.synthetic_roidb(4, seed=6, n_gt=(2, 10))
    it = IT.PrefetchingIter(IT.MNIteratorE2E(roidb, cfg, batch_size=B, n_buffers=5), depth=2, epochs=2,
                            epoch_marker=True)
    stage = IT.InputStage(cfg, DEV, B)
    if kind == "mobilenetv2":
        mc = model_mnv2.MCfg()
        mc.batch_images, mc.bf16 = B, True
        net = model_mnv2.SniperMobileNetV2(mc, device=DEV, seed=3)
    else:
        mc = model.Cfg()
        mc.batch_images, mc.autofocus = B, af
        net = model.SniperResNet101(mc, device=DEV, seed=3)
    tr = trainer.Trainer(mc, device=DEV, net=net, scheduler=None)
    if kind == "resnet101":
        # graphs captured before fit turns the metrics on: enable_metrics then captures the metric graph on its own
        tr.step(synth_batch.make_batch(B, seed=1, device="cpu", pinned=True))
        assert tr.g_up is not None and tr.g_metric is None
    sp = callback.Speedometer(B, 2)
    win = _Window(tr, sp)
    prefix = str(tmp_path / "fit")
    # the window check reads the step's outputs before the next step is enqueued, and the metrics right before the
    # Speedometer resets them
    try:
        tr.fit(it, stage, 2, batch_end_callback=[win, sp], epoch_end_callback=[callback.module_checkpoint(tr, prefix)])
    finally:
        it.close()
    assert win.checked >= 2
    msgs = [r.getMessage() for r in caplog.records]
    assert any(m.startswith("Epoch[1] Time cost=") for m in msgs) and any("Speed:" in m for m in msgs)
    # the epoch-0 checkpoint as main_test.py loads it: `*_test` tensors renamed over the training ones
    arg, aux = checkpoint.load_param(prefix, 1, process=True)
    assert not any(k.endswith("_test") for k in arg)
    b = synth_batch.make_batch(1, seed=2, device=DEV, A=mc.num_anchors, stride=mc.feat_stride)
    if kind == "mobilenetv2":
        tc = model_mnv2.MCfg()
        tc.batch_images, tc.bf16 = 1, True
        test_net = model_mnv2.SniperMobileNetV2(tc, device=DEV, seed=9)
        test_net.load_reference(arg, aux)
        rois, _, cls_prob, _ = test_net.forward_inference(b["data"], b["im_info"])[:4]
        torch.cuda.synchronize()
        assert torch.isfinite(cls_prob).all() and rois.shape[0] > 0
        return
    from sniper_b200 import tester as TS
    tc = model.Cfg()
    tc.batch_images = 2
    test_net = model.SniperResNet101(tc, device=DEV, seed=9)
    test_net.load_reference(arg, aux, allow_missing=True)
    if af:
        test_net.enable_autofocus(arg=arg)       # the trained FocusPixel branch
    else:
        test_net.enable_autofocus(seed=3)
    tcfg = IT.default_config()
    tcfg.TEST.SCALES = [(96, 160), (192, 320), (288, 480)]
    tcfg.TEST.BATCH_IMAGES = [2, 2, 1]
    tcfg.TEST.VALID_RANGES = [(40, -1), (16, 90), (-1, 40)]
    tcfg.TEST.CHIP_HYPERPARAMS = [(3, 0.3, 4), (3, 0.4, 5)]
    rng = np.random.RandomState(2)
    db = [dict(width=W, height=H, image_data=rng.randint(0, 256, (H, W, 3)).astype(np.uint8))
          for (W, H) in ((320, 240), (240, 320), (300, 200))]
    all_boxes, stats = TS.imdb_detection_wrapper(test_net, tcfg, db, detect_backend="device")
    assert len(all_boxes) == 81 and all(len(c) == len(db) for c in all_boxes)
    assert len(stats["scales"]) == 3 and stats["scales"][0]["chips"] > 0
