"""Worker of tests/test_train_ranks_gpu.py.

    python -m torch.distributed.run --nproc-per-node 2 tests/ranks_worker.py train <out> gloo|nccl <train_e2e args>
        tools/train_e2e.py's main on every rank (gloo: joined here, both ranks on cuda:0; nccl: initialised by
        train_e2e on cuda:LOCAL_RANK).  After every epoch each rank dumps its weights, momenta and BatchNorm moving
        statistics to <out>/rank<r>_ep<e>.npz, and it records which epochs it wrote a checkpoint for.
    python tests/ranks_worker.py emulate <out> <train_e2e args>
        the same two-rank training in one process on one GPU: two networks with the same initial weights, each runs
        the captured forward / backward on its rank's slice of the global batch, the gradients are summed g0 + g1
        and each network applies the update.  Dumps <out>/emul<r>_ep<e>.npz."""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import train_e2e as E  # noqa: E402
from sniper_b200 import callback, trainer  # noqa: E402
from sniper_b200 import iterator as IT  # noqa: E402


def dump(path, tr):
    P = tr.net.P
    torch.cuda.synchronize()
    _, aux = tr.net.export_reference()
    np.savez(path, w=P.w.cpu().numpy(), mom=P.mom.cpu().numpy(), **{"aux:" + k: v for k, v in aux.items()})


def train(out, backend, argv):
    import torch.distributed as dist
    rank = int(os.environ["RANK"])
    if backend == "gloo":
        dist.init_process_group("gloo")
        argv = argv + ["--device", "cuda:0"]
    written = []
    save = trainer.Trainer.save_checkpoint

    def recording_save(self, prefix, epoch, *a, **k):
        written.append(epoch)
        return save(self, prefix, epoch, *a, **k)
    trainer.Trainer.save_checkpoint = recording_save
    module_checkpoint = callback.module_checkpoint

    def dumping_checkpoint(tr, prefix, **kw):
        inner = module_checkpoint(tr, prefix, **kw)

        def cb(iter_no, sym=None, arg=None, aux=None):
            dump(os.path.join(out, "rank%d_ep%d.npz" % (rank, iter_no + 1)), tr)
            inner(iter_no, sym, arg, aux)
        return cb
    callback.module_checkpoint = dumping_checkpoint
    res = E.main(argv)
    json.dump(dict(rank=res["rank"], world=res["world_size"], written=written, num_update=res["trainer"].num_update),
              open(os.path.join(out, "rank%d.json" % rank), "w"))
    if backend == "gloo":
        dist.destroy_process_group()


def emulate(out, argv, W=2):
    args = E.parse_args(argv)
    dev = args.device
    cfg = E.config_for(args)
    roidb = E.build_roidb(args, cfg)[0]
    B = args.batch_size
    its = [E.make_iterator(args, cfg, [dict(r) for r in roidb], W, r) for r in range(W)]
    trs = []
    for r in range(W):
        net = E.make_net(args, cfg.dataset.NUM_CLASSES, B, dev)
        net.cfg.roidb_len = len(its[r])
        tr = trainer.Trainer(net.cfg, device=dev, net=net, world_size=W)      # the global batch's lr schedule
        tr.world_size = 1                      # no collective: the gradients are summed below
        trs.append(tr)
    stages = [IT.InputStage(cfg, dev, B) for _ in range(W)]
    steps = 0
    for epoch in range(args.epochs):
        if epoch:
            for it in its:
                it.reset()
        for raws in zip(*its):
            for tr, raw, st in zip(trs, raws, stages):
                batch = st.run(raw)
                if tr.static is None:
                    tr.static = {k: torch.empty_like(v) for k, v in batch.items()}
                for k, v in batch.items():
                    tr.static[k].copy_(v)
                if tr.g_fb is None:
                    tr.capture()
                tr.net.set_lr(tr.next_lr())
                for g in tr.g_fb:
                    g.replay()
            total = trs[0].net.P.g.clone()
            for tr in trs[1:]:
                total += tr.net.P.g
            for tr in trs:
                tr.net.P.g.copy_(total)
                tr.g_up.replay()
            torch.cuda.synchronize()           # the raw batches' buffers are refilled by the next iteration
            steps += 1
        for r, tr in enumerate(trs):
            dump(os.path.join(out, "emul%d_ep%d.npz" % (r, epoch + 1)), tr)
    json.dump(dict(steps=steps), open(os.path.join(out, "emul.json"), "w"))


if __name__ == "__main__":
    if sys.argv[1] == "train":
        train(sys.argv[2], sys.argv[3], sys.argv[4:])
    else:
        emulate(sys.argv[2], sys.argv[3:])
