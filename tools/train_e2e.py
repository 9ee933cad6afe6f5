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
"""
import argparse
import logging
import os
import sys
import time

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
    ap.add_argument("--device", default="cuda:0")
    return ap.parse_args(argv)


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


def train(args, cfg, roidb, batch_end_callback=None, log=logging.getLogger()):
    """The iterator over the roidb (images through host.imread) behind a PrefetchingIter, and Trainer.fit for
    args.epochs epochs with module_checkpoint and batch_end_callback (default: a Speedometer every args.display
    batches).  Returns the trainer."""
    os.makedirs(os.path.dirname(os.path.abspath(args.prefix)), exist_ok=True)
    B = args.batch_size
    it = IT.MNIteratorE2E(roidb, cfg, batch_size=B, image_loader=host.imread, n_buffers=5)
    log.info("the iterator has %d chips", len(it))
    net = make_net(args, cfg.dataset.NUM_CLASSES, B, args.device)
    if args.pretrained:
        load_weights(net, args, args.pretrained, args.pretrained_epoch, log)
    net.cfg.roidb_len = len(it)            # the epoch boundaries of lr_step, as get_optim_params reads them
    if args.lr is not None:
        net.cfg.lr = args.lr
    tr = trainer.Trainer(net.cfg, device=args.device, net=net)
    stage = IT.InputStage(cfg, args.device, B)
    pf = IT.PrefetchingIter(it, depth=2, epochs=args.epochs, epoch_marker=True)
    try:
        if batch_end_callback is None:
            batch_end_callback = callback.Speedometer(B, args.display)
        tr.fit(pf, stage, args.epochs, batch_end_callback=batch_end_callback,
               epoch_end_callback=callback.module_checkpoint(tr, args.prefix))
    finally:
        pf.close()
    return tr


def evaluate(args, cfg, epoch, log=logging.getLogger()):
    """tester.imdb_detection_wrapper on args.test_image_set with `<prefix>-<epoch>.params` (the `*_test` box-regression
    tensors, as main_test.py loads them) and the imdb's evaluation.  Returns (all_boxes, stats)."""
    from sniper_b200 import tester
    imdb = load_data.DATASETS[args.dataset](args.test_image_set, args.root_path, args.dataset_path,
                                            os.path.dirname(os.path.abspath(args.prefix)), device=args.device)
    db = [dict(image=r['image'], width=int(r['width']), height=int(r['height'])) for r in imdb.gt_roidb()]
    net = make_net(args, cfg.dataset.NUM_CLASSES, 1, args.device)
    arg, aux = checkpoint.load_param(args.prefix, epoch, process=True)
    if args.network == "mobilenetv2":
        net.load_reference(arg, aux)
    else:
        net.load_reference(arg, aux, allow_missing=True)
    if args.network == "resnet101_autofocus":
        net.enable_autofocus(arg=arg)
    elif cfg.TEST.AUTO_FOCUS:
        # a network trained without the FocusPixel branch: plain multi-scale inference
        cfg.TEST.AUTO_FOCUS, cfg.TEST.DO_PRUNING = False, [False] * len(cfg.TEST.SCALES)
    all_boxes, stats = tester.imdb_detection_wrapper(net, cfg, db, num_classes=cfg.dataset.NUM_CLASSES,
                                                     device=args.device, imdb=imdb, detect_backend="device",
                                                     image_loader=host.imread)
    log.info("evaluated %s on %d images", args.test_image_set, len(db))
    return all_boxes, stats


def main(argv=None, batch_end_callback=None):
    """Roidb, training and (with --test-image-set) evaluation.  Returns dict(times, bbox_means, bbox_stds, trainer,
    and all_boxes / stats of the evaluation)."""
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(message)s")
    log = logging.getLogger()
    args = parse_args(argv)
    cfg = config_for(args)
    roidb, bbox_means, bbox_stds, times = build_roidb(args, cfg, log)
    times["imread_s_per_image"] = imread_time(roidb)
    log.info("host.imread: %.4f s per image", times["imread_s_per_image"])
    tr = train(args, cfg, roidb, batch_end_callback, log)
    out = dict(times=times, bbox_means=bbox_means, bbox_stds=bbox_stds, trainer=tr)
    if args.test_image_set:
        out["all_boxes"], out["stats"] = evaluate(args, cfg, args.epochs, log)
    return out


if __name__ == "__main__":
    main()
