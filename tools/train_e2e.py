"""main_train.py as a script: a COCO or PASCAL VOC image set on disk -> the training roidb -> Trainer.fit, with the
reference's Speedometer and per-epoch checkpoints; optionally the evaluation of the last checkpoint on a test set.

    python tools/train_e2e.py --dataset PascalVOC --image-set 2007_trainval+2012_trainval --root-path data \\
        --dataset-path data/VOCdevkit --pretrained data/pretrained_model/resnet_mx_101_open --epochs 7 \\
        --prefix output/sniper_voc --test-image-set 2007_test

The roidb is built in main_train.py's order (load_data: proposal roidb of every image set, flipped copies, merge,
filter_roidb, add_bbox_regression_targets); with --proposal-path the RPN proposals there (`<imdb name>_rpn.pkl`, what
tester.imdb_proposal_extraction_wrapper writes) are loaded and TRAIN.USE_NEG_CHIPS is on, otherwise the roidb holds the
GT boxes only.  Images are read from disk by host.imread.  The network starts from `<pretrained>-%04d.params` when given
(checkpoint.load_param, then load_reference(allow_missing=True) as init_weight_rcnn: the layers an ImageNet checkpoint
lacks keep their initialisation), otherwise from the constructor's initialisation.  The time of every roidb stage and of
host.imread per image is logged and returned.

Several GPUs, one process each (the reference trains on every GPU of config.gpus with one iterator of
nGPUs * BATCH_IMAGES chips, main_train.py:44-45, 74):

    python -m torch.distributed.run --nproc-per-node 8 tools/train_e2e.py --batch-size 20 --seed 0 ...

Under torch.distributed.run (WORLD_SIZE > 1) the script joins an already initialised process group or initialises
NCCL on cuda:LOCAL_RANK.  --batch-size stays per GPU; every rank runs MNIteratorE2E over the global batch of
W * batch-size chips with its own rank and the same --seed and trains on its slice, Trainer sums the gradients.  Rank 0
builds the roidb first (it writes the imdb caches), the other ranks then read them, and the ranks' roidbs are compared.
Only rank 0 logs and writes checkpoints, and with --test-image-set rank 0 alone evaluates.  --begin-epoch N resumes
from `<prefix>-N.params` / `.states` on every rank.
"""
import argparse
import logging
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from sniper_b200 import callback, checkpoint, host, load_data, model, model_mnv2, trainer  # noqa: E402
from sniper_b200 import iterator as IT  # noqa: E402

NETWORKS = ("resnet101", "resnet101_autofocus", "mobilenetv2")


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="SNIPER training from an image set on disk (main_train.py)")
    ap.add_argument("--dataset", default="PascalVOC", choices=sorted(load_data.DATASETS))
    ap.add_argument("--image-set", default="2007_trainval+2012_trainval", help="image sets joined by '+'")
    ap.add_argument("--root-path", default="data", help="where the imdb caches go (cache/)")
    ap.add_argument("--dataset-path", default="data/VOCdevkit", help="the VOCdevkit, or COCO's annotations/ + images/")
    ap.add_argument("--proposal-path", default=None, help="RPN proposals for negative chips (TRAIN.USE_NEG_CHIPS)")
    ap.add_argument("--network", default="resnet101", choices=NETWORKS)
    ap.add_argument("--bf16", action="store_true", help="mixed-precision backbone (bf16 operands)")
    ap.add_argument("--batch-size", type=int, default=16, help="chips per step (TRAIN.BATCH_IMAGES)")
    ap.add_argument("--epochs", type=int, default=7, help="TRAIN.end_epoch")
    ap.add_argument("--lr", type=float, default=None, help="base learning rate (default: the config's)")
    ap.add_argument("--pretrained", default=None, help="checkpoint prefix of the initial weights")
    ap.add_argument("--pretrained-epoch", type=int, default=0)
    ap.add_argument("--prefix", default="output/SNIPER", help="checkpoint prefix (<prefix>-%%04d.params / .states)")
    ap.add_argument("--display", type=int, default=100, help="Speedometer period in batches")
    ap.add_argument("--test-image-set", default=None, help="after training, evaluate the last checkpoint on this set")
    ap.add_argument("--device", default="cuda:0", help="the GPU (under torch.distributed.run with NCCL: cuda:LOCAL_RANK)")
    ap.add_argument("--seed", type=int, default=None,
                    help="seed of the iterator's draws, the same on every rank (default: the global np.random with one "
                         "process, 0 with several)")
    ap.add_argument("--plan-backend", default="host", choices=("host", "device"),
                    help="where each epoch's chip plan (chips, box assignment, negative chips) is computed; the device "
                         "plan is byte-equal to the host one")
    ap.add_argument("--begin-epoch", type=int, default=0,
                    help="resume: load <prefix>-<N>.params / .states and train epochs N+1 .. --epochs")
    return ap.parse_args(argv)


def init_distributed(args):
    """-> (world size, rank).  Joins an initialised process group; otherwise, under a launcher with WORLD_SIZE > 1,
    initialises NCCL on cuda:LOCAL_RANK (args.device is set to it).  One process: (1, 0), nothing initialised."""
    dist = torch.distributed
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(), dist.get_rank()
    if int(os.environ.get("WORLD_SIZE", "1")) <= 1:
        return 1, 0
    local = int(os.environ.get("LOCAL_RANK", "0"))
    args.device = "cuda:%d" % local
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    return dist.get_world_size(), dist.get_rank()


def _same_on_all_ranks(value, what, world):
    """Collective: raises ValueError on every rank unless `value` is equal on all of them."""
    if world <= 1:
        return
    got = [None] * world
    torch.distributed.all_gather_object(got, value)
    if any(v != got[0] for v in got):
        raise ValueError("the ranks' %s differ: %s" % (what, ", ".join("rank %d: %r" % (r, v) for r, v in enumerate(got))))


def config_for(args):
    """iterator.default_config of the dataset and network, with main_train.py's COCO scale rule applied."""
    cfg = IT.default_config(neg=args.proposal_path is not None, autofocus=args.network == "resnet101_autofocus",
                            network="mobilenetv2" if args.network == "mobilenetv2" else "resnet101",
                            dataset="pascal_voc" if args.dataset == "PascalVOC" else "coco")
    load_data.paper_train_scales(cfg)
    return cfg


def build_roidb(args, cfg, log=logging.getLogger()):
    """main_train.py:54-66.  Returns (roidb, bbox_means, bbox_stds, times): times holds the seconds of every stage
    summed over the image sets (gt_s, rpn_s: the proposal file, its device NMS and the GT overlaps; flip_s), of the
    merge, the filter and the targets, and the image count before and after the filter."""
    times = dict(gt_s=0.0, rpn_s=0.0, flip_s=0.0)
    roidbs = []
    for image_set in args.image_set.split('+'):
        t = {}
        roidbs.append(load_data.load_proposal_roidb(args.dataset, image_set, args.root_path, args.dataset_path,
                                                    result_path=os.path.dirname(os.path.abspath(args.prefix)),
                                                    flip=cfg.TRAIN.FLIP, proposal_path=args.proposal_path,
                                                    only_gt=not cfg.TRAIN.USE_NEG_CHIPS, device=args.device, times=t))
        for k in t:
            times[k] += t[k]
    t0 = time.time()
    roidb = load_data.merge_roidb(roidbs)
    times["entries"] = len(roidb)
    t1 = time.time()
    roidb = load_data.filter_roidb(roidb, cfg)
    t2 = time.time()
    bbox_means, bbox_stds = load_data.add_bbox_regression_targets(roidb, cfg)
    times.update(merge_s=t1 - t0, filter_s=t2 - t1, targets_s=time.time() - t2, entries_kept=len(roidb))
    log.info("roidb: %d entries (%d after filter_roidb); seconds: %s", times["entries"], len(roidb),
             ", ".join("%s %.3f" % (k, v) for k, v in times.items() if k.endswith("_s")))
    return roidb, bbox_means, bbox_stds, times


def make_net(args, num_classes, batch_images, device):
    if args.network == "mobilenetv2":
        c = model_mnv2.MCfg()
        c.num_classes, c.batch_images, c.bf16 = num_classes, batch_images, args.bf16
        return model_mnv2.SniperMobileNetV2(c, device=device)
    c = model.Cfg()
    c.num_classes, c.batch_images, c.bf16 = num_classes, batch_images, args.bf16
    c.autofocus = args.network == "resnet101_autofocus"
    return model.SniperResNet101(c, device=device)


def load_weights(net, args, prefix, epoch, log=logging.getLogger()):
    arg, aux = checkpoint.load_param(prefix, epoch)
    if args.network == "mobilenetv2":
        net.load_reference(arg, aux)
    else:
        skipped = net.load_reference(arg, aux, allow_missing=True)
        log.info("initialised from %s-%04d.params; %d layers not in it keep their initialisation", prefix, epoch,
                 len(skipped))


def imread_time(roidb, n=20):
    """Seconds per image of host.imread over the first n distinct image files of the roidb."""
    paths = list(dict.fromkeys(r['image'] for r in roidb))[:n]
    t0 = time.time()
    for p in paths:
        host.imread(p)
    return (time.time() - t0) / max(len(paths), 1)


def make_iterator(args, cfg, roidb, world=1, rank=0):
    """MNIteratorE2E over the global batch of world * args.batch_size chips; with several ranks, this rank's slice of
    it.  A resumed run (--begin-epoch N) skips the plans of the N epochs already trained."""
    seed = args.seed if args.seed is not None or world == 1 else 0
    it = IT.MNIteratorE2E(roidb, cfg, batch_size=world * args.batch_size, nGPUs=world, image_loader=host.imread,
                          n_buffers=5, rank=None if world == 1 else rank, seed=seed,
                          plan_backend=getattr(args, "plan_backend", "host"),
                          device=args.device if getattr(args, "plan_backend", "host") == "device" else None)
    for _ in range(args.begin_epoch):
        it.reset()
    return it


def train(args, cfg, roidb, batch_end_callback=None, log=logging.getLogger(), world=1, rank=0):
    """The iterator over the roidb (images through host.imread) behind a PrefetchingIter, and Trainer.fit for
    args.epochs epochs with module_checkpoint and batch_end_callback (default: a Speedometer every args.display
    batches, counting the chips of all ranks).  Returns the trainer."""
    os.makedirs(os.path.dirname(os.path.abspath(args.prefix)), exist_ok=True)
    B = args.batch_size
    it = make_iterator(args, cfg, roidb, world, rank)
    log.info("the iterator has %d chips", len(it))
    net = make_net(args, cfg.dataset.NUM_CLASSES, B, args.device)
    if args.begin_epoch > 0:
        arg, aux = checkpoint.load_param(args.prefix, args.begin_epoch)
        net.load_reference(arg, aux)
        log.info("resuming from %s-%04d.params", args.prefix, args.begin_epoch)
    elif args.pretrained:
        load_weights(net, args, args.pretrained, args.pretrained_epoch, log)
    net.cfg.roidb_len = len(it)            # the epoch boundaries of lr_step, as get_optim_params reads them
    if args.lr is not None:
        net.cfg.lr = args.lr
    tr = trainer.Trainer(net.cfg, device=args.device, net=net, world_size=world)
    if args.begin_epoch > 0:
        tr.load_optimizer_states("%s-%04d.states" % (args.prefix, args.begin_epoch))
    stage = IT.InputStage(cfg, args.device, B)
    pf = IT.PrefetchingIter(it, depth=2, epochs=args.epochs - args.begin_epoch, epoch_marker=True)
    try:
        if batch_end_callback is None:
            batch_end_callback = callback.Speedometer(world * B, args.display)
        tr.fit(pf, stage, args.epochs, begin_epoch=args.begin_epoch, batch_end_callback=batch_end_callback,
               epoch_end_callback=callback.module_checkpoint(tr, args.prefix))
    finally:
        pf.close()
    return tr


def load_test_net(args, cfg, epoch):
    """The network of `<prefix>-<epoch>.params` for inference, with the `*_test` box-regression tensors as main_test.py
    loads them (checkpoint.load_param(process=True)).  For a network without the FocusPixel branch, cfg.TEST's
    AUTO_FOCUS / DO_PRUNING are turned off: plain multi-scale inference."""
    net = make_net(args, cfg.dataset.NUM_CLASSES, 1, args.device)
    arg, aux = checkpoint.load_param(args.prefix, epoch, process=True)
    if args.network == "mobilenetv2":
        net.load_reference(arg, aux)
    else:
        net.load_reference(arg, aux, allow_missing=True)
    if args.network == "resnet101_autofocus":
        net.enable_autofocus(arg=arg)
    elif cfg.TEST.AUTO_FOCUS:
        cfg.TEST.AUTO_FOCUS, cfg.TEST.DO_PRUNING = False, [False] * len(cfg.TEST.SCALES)
    return net


def evaluate(args, cfg, epoch, log=logging.getLogger()):
    """tester.imdb_detection_wrapper on args.test_image_set with `<prefix>-<epoch>.params` (the `*_test` box-regression
    tensors, as main_test.py loads them) and the imdb's evaluation.  Returns (all_boxes, stats)."""
    from sniper_b200 import tester
    imdb = load_data.DATASETS[args.dataset](args.test_image_set, args.root_path, args.dataset_path,
                                            os.path.dirname(os.path.abspath(args.prefix)), device=args.device)
    db = [dict(image=r['image'], width=int(r['width']), height=int(r['height'])) for r in imdb.gt_roidb()]
    net = load_test_net(args, cfg, epoch)
    all_boxes, stats = tester.imdb_detection_wrapper(net, cfg, db, num_classes=cfg.dataset.NUM_CLASSES,
                                                     device=args.device, imdb=imdb, detect_backend="device",
                                                     image_loader=host.imread)
    log.info("evaluated %s on %d images", args.test_image_set, len(db))
    return all_boxes, stats


def main(argv=None, batch_end_callback=None):
    """Roidb, training and (with --test-image-set) evaluation on rank 0.  Returns dict(times, bbox_means, bbox_stds,
    trainer, world_size, rank, and all_boxes / stats of the evaluation).  A process group this call initialised is
    destroyed before it returns."""
    args = parse_args(argv)
    dist = torch.distributed
    owned = not (dist.is_available() and dist.is_initialized())
    world, rank = init_distributed(args)
    logging.basicConfig(level=logging.INFO if rank == 0 else logging.WARNING, format="%(asctime)s %(message)s")
    log = logging.getLogger()
    try:
        cfg = config_for(args)
        # rank 0 first: it writes the imdb caches and the proposals' _rpn_after_nms.pkl the other ranks then read
        if rank == 0:
            roidb, bbox_means, bbox_stds, times = build_roidb(args, cfg, log)
        if world > 1:
            dist.barrier()
            if rank != 0:
                roidb, bbox_means, bbox_stds, times = build_roidb(args, cfg, log)
            _same_on_all_ranks(IT.roidb_digest(roidb), "training roidbs", world)
        times["imread_s_per_image"] = imread_time(roidb)
        log.info("host.imread: %.4f s per image", times["imread_s_per_image"])
        tr = train(args, cfg, roidb, batch_end_callback, log, world, rank)
        out = dict(times=times, bbox_means=bbox_means, bbox_stds=bbox_stds, trainer=tr, world_size=world, rank=rank)
        if world > 1:
            dist.barrier()                 # rank 0 has written the last checkpoint
        if args.test_image_set and rank == 0:
            out["all_boxes"], out["stats"] = evaluate(args, cfg, args.epochs, log)
        return out
    finally:
        if owned and world > 1:
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
