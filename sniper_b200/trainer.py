"""Training-step driver: the `Module.forward_backward` / `update` / `update_metric` inner loop of
BaseModule.fit (SNIPER-mxnet/python/mxnet/module/base_module.py:505-535) for the SNIPER graph.

One process per GPU.  Per step: pinned host batch -> H2D (on a copy stream, one step ahead when the caller names the
next batch: `step(batch, prefetch=next_batch)`, as MNIteratorE2E's prefetch threads do), one CUDA-graph replay of
forward+backward, ONE NCCL all-reduce over the flat gradient bucket (replaces the per-key kvstore
push/pull, model.py:126-136 / comm.h:433-553; sum without 1/N as rescale_grad=1.0, utils.py:30,37), one
CUDA-graph replay of the fused SGD-momentum update, D2H of the four loss scalars (what the reference's
metrics read with asnumpy(), lib/train_utils/metric.py:109-125).

`fit` is BaseModule.fit's epoch loop (base_module.py:500-550) on top of that step.  It turns on the device metrics
(`metrics=True`): one `sniper_train_metric_accum` launch per step, after the update, accumulates the reference's
training metrics on the device, so a step needs no host synchronisation and the metrics are read only when printed.
"""
import logging
import time
from collections import namedtuple

import numpy as np
import torch

from . import checkpoint, lr_scheduler, metric, model, ops

# mxnet.model.BatchEndParam (SNIPER-mxnet/python/mxnet/model.py:51-56)
BatchEndParam = namedtuple("BatchEndParams", ["epoch", "nbatch", "eval_metric", "locals"])


def check_plan(digest, world_size, epoch=None):
    """Collective: every rank passes the plan digest of its epoch's first raw batch (`RawBatch.plan_digest`, None when
    the iterator gives none).  Raises ValueError on every rank, naming the ranks, when the ranks' plans differ, so
    that no rank goes on into a collective the others never reach.  Digests that are None on every rank are not
    checked."""
    if world_size <= 1:
        return
    got = [None] * world_size
    torch.distributed.all_gather_object(got, None if digest is None else int(digest))
    if all(d is None for d in got) or all(d == got[0] for d in got):
        return
    groups = {}
    for r, d in enumerate(got):
        groups.setdefault(d, []).append(r)
    raise ValueError("%sthe ranks' epoch plans differ (different iterator seeds, roidbs or configs?): %s" % (
        "" if epoch is None else "epoch %d: " % epoch,
        "; ".join("ranks %s: %s" % (rs, "no digest" if d is None else "%016x" % d) for d, rs in groups.items())))


class Trainer:
    def __init__(self, cfg=None, device="cuda:0", world_size=1, use_graph=True, seed=5, deform_offset_std=0.0,
                 scheduler="config", net=None, metrics=False):
        """scheduler: "config" = the reference's WarmupMultiBatchScheduler built from cfg (lr, lr_step, warmup*), None =
        constant cfg.lr, or any callable num_update -> lr.  net: an already constructed network exposing the same
        surface as model.SniperResNet101 (P, fb_phases, forward_backward, train_bns, set_lr, update), e.g.
        model_mnv2.SniperMobileNetV2; default: the ResNet-101 graph built from cfg.  metrics: accumulate the training
        metrics on the device after every step (`metric_acc`; `fit` turns this on)."""
        self.cfg = cfg or (net.cfg if net is not None else model.Cfg())
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)
        self.world_size = world_size
        self._works = []
        self.net = net if net is not None else model.SniperResNet101(self.cfg, device=self.device, seed=seed,
                                                                     deform_offset_std=deform_offset_std)
        self.use_graph = use_graph
        self.static = None
        self.g_fb = None
        self.g_up = None
        self.out = None
        self.loss_host = torch.zeros(8).pin_memory()
        self.launches_per_step = 0
        # input pipeline: two device staging sets filled by a copy stream while the previous step computes
        self.copy_stream = torch.cuda.Stream(device=self.device)
        self.stage = [None, None]
        self.stage_ready = [None, None]      # event: H2D into stage[i] finished
        self.stage_free = [None, None]       # event: the step that consumed stage[i] has copied it out
        self.stage_owner = [None, None]      # the host batch object sitting in stage[i] (kept alive: identity match)
        self.next_stage = 0
        # optimizer state of mxnet.optimizer.SGD that lives on the host: update count and LR schedule
        self.num_update = 0
        if scheduler == "config":
            c = self.cfg
            scheduler = lr_scheduler.from_config(lr=c.lr, lr_step=getattr(c, "lr_step", "5.33"),
                                                 lr_factor=getattr(c, "lr_factor", 0.1), warmup=getattr(c, "warmup", True),
                                                 warmup_lr=getattr(c, "warmup_lr", 0.0005),
                                                 warmup_step=getattr(c, "warmup_step", 1000),
                                                 roidb_len=getattr(c, "roidb_len", None),
                                                 batch_size=getattr(c, "batch_images", 16) * world_size)
        self.scheduler = scheduler
        self.lr = self.cfg.lr
        self.metric_acc = None
        self.g_metric = None
        if metrics:
            self.enable_metrics()

    def enable_metrics(self):
        """Adds the metric launch to every following step (and, with graphs, a small graph replayed after the update)."""
        if self.metric_acc is None:
            self.metric_acc = metric.MetricAccumulator(self.device, self.world_size)
            if self.g_up is not None:
                self._capture_metric(torch.cuda.graph_pool_handle())
        return self.metric_acc

    def _metric_launch(self, out, acc=None):
        """The step's metric terms into the accumulator: RPN probabilities against the batch's anchor labels, R-CNN
        class probabilities against MultiProposalTarget's labels, and (AutoFocus) the FocusPixel softmax."""
        net = self.net
        if not getattr(net, "rcnn_valid_counted", True):
            ops.count_valid(out["label"], net.cnt_buf[1:2])      # a net whose R-CNN loss does not count its rows
        ops.train_metric_accum(out["rpn_cls_prob"], self.static["label"], net.cfg.num_anchors, out["cls_prob"],
                               out["label"], net.cnt_buf, net.loss_buf, self.metric_acc.buf if acc is None else acc,
                               self.metric_acc.workspace, af_prob=out.get("cls_scale_prob"),
                               af_label=out.get("scale_label"))

    def _capture_metric(self, pool):
        # one eager launch first loads the kernel outside capture; its sum goes to a scratch accumulator and is dropped
        self._metric_launch(self.out, acc=torch.zeros_like(self.metric_acc.buf))
        torch.cuda.synchronize()
        self.g_metric = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_metric, pool=pool):
            self._metric_launch(self.out)
        torch.cuda.synchronize()

    def next_lr(self, lr=None):
        """mxnet.optimizer: `_update_count` then `_get_lr` -> scheduler(num_update) with the incremented count."""
        self.num_update += 1
        if lr is None:
            lr = self.scheduler(self.num_update) if self.scheduler is not None else self.cfg.lr
        self.lr = float(lr)
        return self.lr

    # ---- device-resident step (inputs already in HBM)
    def _alloc_static(self, batch):
        self.static = {k: torch.empty_like(v, device=self.device) for k, v in batch.items()}

    def load(self, host_batch):
        """H2D of one chip batch (pinned host tensors) into the static device buffers."""
        if self.static is None:
            self._alloc_static(host_batch)
        for k, v in host_batch.items():
            self.static[k].copy_(v, non_blocking=True)

    def prefetch(self, host_batch):
        """Starts the H2D of a FUTURE batch on the copy stream (overlaps the step in flight)."""
        i = self.next_stage
        self.next_stage ^= 1
        if self.stage[i] is None:
            self.stage[i] = {k: torch.empty_like(v, device=self.device) for k, v in host_batch.items()}
        if self.stage_free[i] is not None:
            self.copy_stream.wait_event(self.stage_free[i])
        with torch.cuda.stream(self.copy_stream):
            for k, v in host_batch.items():
                self.stage[i][k].copy_(v, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self.stage_ready[i] = ev
        self.stage_owner[i] = host_batch

    def _load_or_take(self, host_batch):
        """Brings `host_batch` into the static buffers: from its staging set if it was prefetched, else by H2D now."""
        for i in (0, 1):
            if self.stage_owner[i] is host_batch and self.stage_ready[i] is not None:
                if self.static is None:
                    self._alloc_static(host_batch)
                cur = torch.cuda.current_stream()
                cur.wait_event(self.stage_ready[i])
                for k in self.static:
                    self.static[k].copy_(self.stage[i][k], non_blocking=True)     # D2D, ~25 us
                ev = torch.cuda.Event()
                ev.record(cur)
                self.stage_free[i] = ev
                self.stage_owner[i] = None
                return
        self.load(host_batch)

    def _allreduce(self):
        """The whole gradient buffer in one collective (eager / warm-up path)."""
        if self.world_size > 1:
            torch.distributed.all_reduce(self.net.P.g, op=torch.distributed.ReduceOp.SUM)

    def _allreduce_bucket(self, k):
        """Starts the sum of gradient bucket k over the ranks on NCCL's own stream (it first waits for everything
        enqueued so far on the current stream, i.e. the phase that produced the bucket) and returns at once, so the next
        backward phase overlaps the transfer.  No 1/N: rescale_grad = 1.0 (lib/train_utils/utils.py:30,37)."""
        if self.world_size > 1:
            a, b = self.net.P.bucket_ranges[k]
            self._works.append(torch.distributed.all_reduce(self.net.P.g[a:b], op=torch.distributed.ReduceOp.SUM,
                                                            async_op=True))

    def _allreduce_finish(self):
        for w in self._works:
            w.wait()                              # the current stream waits for the collective
        self._works = []

    def export_reference(self):
        """net.export_reference() as a checkpoint holds it.  With several ranks this is a collective: every auxiliary
        state (the BatchNorm moving statistics, which each rank updates from its own chips) is averaged over the ranks as
        DataParallelExecutorGroup.get_params does (module/executor_group.py:415-420): float32, summed in rank order
        starting from rank 0's value, then divided by the number of ranks.  The weights are identical on every rank."""
        arg, aux = self.net.export_reference()
        if self.world_size <= 1 or not aux:
            return arg, aux
        names = sorted(aux)
        flat = torch.from_numpy(np.concatenate([np.ascontiguousarray(aux[k], np.float32).ravel() for k in names]))
        if torch.distributed.get_backend() == "nccl":
            flat = flat.to(self.device)
        got = [torch.empty_like(flat) for _ in range(self.world_size)]
        torch.distributed.all_gather(got, flat)
        got = [g.cpu().numpy() for g in got]
        total = got[0].copy()
        for g in got[1:]:
            total += g
        total /= np.float32(self.world_size)
        off = 0
        for k in names:
            n = aux[k].size
            aux[k] = total[off:off + n].reshape(aux[k].shape).copy()
            off += n
        return arg, aux

    def _snapshot(self):
        P = self.net.P
        bns = self.net.train_bns()
        return (P.w.clone(), P.mom.clone(), [(b.st.moving_mean.clone(), b.st.moving_var.clone()) for b in bns])

    def _restore(self, snap):
        P = self.net.P
        P.w.copy_(snap[0])
        P.mom.copy_(snap[1])
        for b, (m, v) in zip(self.net.train_bns(), snap[2]):
            b.st.moving_mean.copy_(m)
            b.st.moving_var.copy_(v)
        # the warm-up's lr-0 updates still move the weights by the momentum (non-zero after a resume), and the bf16
        # copies with them: rebuild those from the restored fp32 masters
        P.sync_lowp()

    def capture(self):
        """Warm up eagerly, then capture forward+backward and the optimizer update as two CUDA graphs.  The warm-up runs
        complete training steps on whatever sits in the static buffers; weights, momentum and the BN moving statistics
        are snapshotted before and restored afterwards, so capture() leaves the model exactly as it found it (a freshly
        loaded checkpoint is not disturbed and the first step() applies ONE update, like the reference's)."""
        snap = self._snapshot()
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self.net.set_lr(0.0)
            for _ in range(2):
                ops.reset_launch_count()
                self.out = self.net.forward_backward(self.static)
                self._allreduce()
                self.net.update()
                self.launches_per_step = ops.launch_count()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self._restore(snap)
        if not self.use_graph:
            return
        # forward + backward as one CUDA graph per gradient bucket (model.fb_phases), sharing one memory pool: between
        # the replays the trainer starts the bucket's all-reduce, which then runs under the next phase's kernels
        pool = torch.cuda.graph_pool_handle()
        self.g_fb = []
        phases = self.net.fb_phases(self.static)
        for _ in range(getattr(self.net, "n_phases", 3)):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=pool):
                self.out = next(phases)
            self.g_fb.append(g)
        self.g_up = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_up, pool=pool):
            self.net.update()
        torch.cuda.synchronize()
        if self.metric_acc is not None:
            self._capture_metric(pool)

    def step_device(self, lr=None):
        """One training step on the batch currently in the static buffers.  The learning rate comes from the schedule
        (or `lr`) and reaches the captured update graph through the device hyper-parameter buffer."""
        self.net.set_lr(self.next_lr(lr))
        if self.g_fb is not None:
            for k, g in enumerate(self.g_fb):
                g.replay()
                self._allreduce_bucket(k)
            self._allreduce_finish()
            self.g_up.replay()
            if self.g_metric is not None:
                self.g_metric.replay()
        else:
            self.out = self.net.forward_backward(self.static, on_bucket=self._allreduce_bucket)
            self._allreduce_finish()
            self.net.update()
            if self.metric_acc is not None:
                self._metric_launch(self.out)
        return self.out

    # ---- public end-to-end step from the iterator's raw batch (uint8 source rectangles + chip tables)
    def step_raw(self, raw, input_stage, lr=None):
        """One training step on a `iterator.RawBatch`: H2D of the raw bytes, GPU input stage (resize / mean / flip,
        anchor matching, label subsampling), forward + backward + all-reduce + update, D2H of the losses."""
        return self._losses(self._enqueue_raw(raw, input_stage, lr))

    def _enqueue_raw(self, raw, input_stage, lr):
        batch = input_stage.run(raw)
        if self.static is None:
            self.static = {k: torch.empty_like(v) for k, v in batch.items()}
        for k, v in batch.items():
            self.static[k].copy_(v, non_blocking=True)
        if self.g_fb is None and self.use_graph:
            self.capture()
        return self.step_device(lr)

    def step_raw_async(self, raw, input_stage, lr=None):
        """step_raw without the loss read-back: enqueues the step (and, with metrics on, its metric launch) and returns
        at once with an event that completes with the step.  The raw batch's pinned buffers are read by asynchronous
        H2D copies until then."""
        self._enqueue_raw(raw, input_stage, lr)
        done = torch.cuda.Event()
        done.record()
        return done

    def _losses(self, out):
        """D2H of the step's loss buffer (one 32-byte copy) -> the metric values; an AutoFocus net adds the cls_scale_prob
        loss sum and AutoFocusAccMetric (lib/train_utils/metric.py:50-72: argmax hits over non-ignored FocusPixels)."""
        self.loss_host.copy_(out["losses"], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        h = self.loss_host
        r = {"rpn_cls_loss": float(h[0]), "rpn_bbox_loss": float(h[1]), "rcnn_cls_loss": float(h[2]),
             "rcnn_bbox_loss": float(h[3]), "lr": self.lr}
        if getattr(self.net.cfg, "autofocus", False):
            r["autofocus_cls_loss"] = float(h[4])
            r["autofocus_acc"] = float(h[5]) / max(float(h[6]), 1.0)
        return r

    # ---- public end-to-end step: host batch in, host losses out
    def step(self, host_batch, prefetch=None, lr=None):
        """One training step on `host_batch` (pinned host tensors) -> host loss scalars.  `prefetch`: the batch of the
        NEXT call; its H2D copy is issued now on the copy stream and overlaps this step's compute.  `lr` overrides the
        schedule for this update."""
        self._load_or_take(host_batch)
        if prefetch is not None:
            self.prefetch(prefetch)
        if self.g_fb is None and self.use_graph:
            self.capture()
        return self._losses(self.step_device(lr))

    # ---- checkpoints (Module.save_checkpoint / load_optimizer_states, module.py:160-180, 775-805)
    def save_checkpoint(self, prefix, epoch, save_optimizer_states=False, arg_params=None, aux_params=None):
        """`<prefix>-%04d.params` through checkpoint.save_checkpoint (with the `*_test` box-regression tensors), the
        bound Symbol's `<prefix>-symbol.json` when the net came from one, and `<prefix>-%04d.states` (momenta and the
        update count) when asked.  arg_params / aux_params: what `export_reference()` returned (fit passes them to its
        epoch-end callbacks); without them it is called here, which with several ranks is a collective."""
        arg, aux = (arg_params, aux_params) if arg_params is not None else self.export_reference()
        sym = getattr(self.net, "symbol", None)
        if sym is not None:
            sym.save("%s-symbol.json" % prefix)
        checkpoint.save_checkpoint(prefix, epoch, arg, aux)
        if save_optimizer_states:
            checkpoint.save_optimizer_states("%s-%04d.states" % (prefix, epoch), self.net, self.num_update)

    def load_optimizer_states(self, fname):
        """Momenta and update count of a `.states` file written by save_checkpoint: the next step continues the run
        (the learning-rate schedule follows num_update)."""
        self.num_update = checkpoint.load_optimizer_states(fname, self.net)

    # ---- the epoch loop
    def fit(self, train_iter, input_stage, num_epoch, begin_epoch=0, eval_metric=None, batch_end_callback=None,
            epoch_end_callback=None):
        """BaseModule.fit (SNIPER-mxnet/python/mxnet/module/base_module.py:500-550) over raw batches.

        train_iter: an `iterator.PrefetchingIter(..., epoch_marker=True)` (an epoch ends at its marker: the chip count
        changes from epoch to epoch with the negative-chip draw), or any iterator of raw batches that ends each epoch
        with StopIteration and has `reset()`.  eval_metric: a `metric` object (default: main_train.py's composite);
        it is bound to this trainer's device accumulator.  batch_end_callback(BatchEndParam) after every step,
        epoch_end_callback(epoch, symbol, arg_params, aux_params) after every epoch; lists are accepted.

        The host runs at most one step ahead of the device: before step i+1 is enqueued (and before its raw batch is
        taken from the iterator) step i-1 has completed, so at most two raw batches are read by in-flight H2D copies.
        With several ranks every rank must call fit with its own `MNIteratorE2E(batch_size=W*B, nGPUs=W, rank=r,
        seed=s)`, the same seed on every rank: each rank then takes its slice of every global batch, and all ranks
        have the same epoch length.  At the first batch of every epoch fit all-gathers the batch's plan digest (on
        this thread, so the collectives keep one order on every rank) and raises ValueError on every rank if they
        differ.  Metric reads are collective, and only rank 0 logs.  The arg / aux params passed to
        epoch_end_callback come from `export_reference()` (on every rank): the BatchNorm moving statistics averaged
        over the ranks, as the reference's checkpoint holds them.  Verified with two ranks sharing one GPU over gloo
        (tests/test_train_ranks_gpu.py, TF32 and bf16): after every epoch the weights and momenta are identical on both
        ranks and byte-equal to a one-process emulation of the two slices with the gradients summed, and a resumed run
        ends byte-equal to an uninterrupted one.  The test's NCCL variant needs two GPUs."""
        from . import iterator
        if isinstance(train_iter, iterator.PrefetchingIter) and not train_iter.epoch_marker:
            raise ValueError("fit: a PrefetchingIter needs epoch_marker=True (it would run one endless epoch)")
        if isinstance(train_iter, iterator.PrefetchingIter) and hasattr(train_iter.it, "_buffers"):
            need = train_iter.q.maxsize + 3
            if len(train_iter.it._buffers) < need:
                raise ValueError("fit: the iterator owns %d raw buffers; with prefetch depth %d it needs %d (two "
                                 "batches in flight, see iterator.RawBatch)" % (len(train_iter.it._buffers),
                                                                                train_iter.q.maxsize, need))
        acc = self.enable_metrics()
        if eval_metric is None:
            eval_metric = metric.default_metrics(bool(getattr(self.net.cfg, "autofocus", False)))
        eval_metric.bind(acc)
        rank0 = self.world_size == 1 or torch.distributed.get_rank() == 0
        log = logging.getLogger()
        as_list = lambda c: [] if c is None else (c if isinstance(c, (list, tuple)) else [c])
        marker = getattr(iterator, "EPOCH_END", None)

        def fetch(it):
            try:
                b = next(it)
            except StopIteration:
                return None
            return None if b is marker else b

        for epoch in range(begin_epoch, num_epoch):
            tic = time.time()
            eval_metric.reset()
            nbatch = 0
            it = iter(train_iter)
            done = [None, None]                  # completion events of the last two steps enqueued
            next_raw = fetch(it)
            check_plan(getattr(next_raw, "plan_digest", None), self.world_size, epoch)
            eval_name_vals = []
            while next_raw is not None:
                raw = next_raw
                done = [done[1], self.step_raw_async(raw, input_stage)]
                if done[0] is not None:
                    done[0].synchronize()        # step i-1 done: its raw batch may be refilled
                next_raw = fetch(it)
                if next_raw is None:
                    eval_name_vals = eval_metric.get_name_value()
                param = BatchEndParam(epoch=epoch, nbatch=nbatch, eval_metric=eval_metric, locals=locals())
                for cb in as_list(batch_end_callback):
                    cb(param)
                nbatch += 1
            if done[1] is not None:
                done[1].synchronize()
            if rank0:
                for name, val in eval_name_vals:
                    log.info("Epoch[%d] Train-%s=%f", epoch, name, val)
                log.info("Epoch[%d] Time cost=%.3f", epoch, time.time() - tic)
            if epoch_end_callback is not None:
                arg, aux = self.export_reference()
                for cb in as_list(epoch_end_callback):
                    cb(epoch, getattr(self.net, "symbol", None), arg, aux)
            if not isinstance(train_iter, iterator.PrefetchingIter):
                train_iter.reset()
