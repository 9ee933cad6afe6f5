"""main_test.py as a script: a checkpoint -> detections on a COCO or PASCAL VOC image set on disk and the imdb's
evaluation, or (--extract-proposals) the RPN proposals of every image for negative-chip mining and their recall.

    python tools/test_e2e.py --dataset PascalVOC --image-set 2007_test --root-path data \\
        --dataset-path data/VOCdevkit --prefix output/sniper_voc --epoch 7

    python tools/test_e2e.py --extract-proposals --proposal-save-path data/computed_proposals \\
        --image-set 2007_trainval+2012_trainval --prefix output/sniper_neg_proposals --epoch 2 ...

The network is `<prefix>-<epoch>.params` with the `*_test` box-regression tensors (train_e2e.load_test_net).  Image
sets joined by '+' are run one after the other, each with its own evaluation, or its own `<DATASET>_<set>_rpn.pkl`
under --proposal-save-path (tester.proposal_file_name), as scripts/train_neg_props_and_sniper.sh loops over the
training sets.  Images are read from disk by host.imread.

--concurrent-jobs J is TEST.CONCURRENT_JOBS: the images are split into J blocks and each block runs the test pipeline
on its own (tester.imdb_detection_wrapper).  Several GPUs, one process each:

    python -m torch.distributed.run --nproc-per-node 8 tools/test_e2e.py ...

Under torch.distributed.run the script joins an already initialised process group or initialises NCCL on
cuda:LOCAL_RANK (train_e2e.init_distributed).  J defaults to the world size; job j runs on rank j mod W, which reads
only its own images.  Rank 0 builds the imdb caches first, the other ranks then read them.  Rank 0 alone logs, merges
the jobs, evaluates and writes files.
"""
import argparse
import logging
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from sniper_b200 import host, load_data, tester  # noqa: E402
from sniper_b200 import iterator as IT  # noqa: E402
from train_e2e import NETWORKS, init_distributed, load_test_net  # noqa: E402


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="SNIPER inference on an image set on disk (main_test.py)")
    ap.add_argument("--dataset", default="PascalVOC", choices=sorted(load_data.DATASETS))
    ap.add_argument("--image-set", default="2007_test", help="image sets joined by '+', run one after the other")
    ap.add_argument("--root-path", default="data", help="where the imdb caches go (cache/)")
    ap.add_argument("--dataset-path", default="data/VOCdevkit", help="the VOCdevkit, or COCO's annotations/ + images/")
    ap.add_argument("--prefix", default="output/SNIPER", help="checkpoint prefix (<prefix>-%%04d.params); the "
                    "evaluation's result files go to its directory")
    ap.add_argument("--epoch", type=int, default=7, help="TEST.TEST_EPOCH")
    ap.add_argument("--network", default="resnet101", choices=NETWORKS)
    ap.add_argument("--bf16", action="store_true", help="mixed-precision backbone (bf16 operands)")
    ap.add_argument("--extract-proposals", action="store_true", help="TEST.EXTRACT_PROPOSALS")
    ap.add_argument("--proposal-save-path", default="output/proposals", help="TEST.PROPOSAL_SAVE_PATH")
    ap.add_argument("--concurrent-jobs", type=int, default=None, help="TEST.CONCURRENT_JOBS (default: the world size)")
    ap.add_argument("--detect-backend", default="device", choices=("device", "host"),
                    help="where the detections are decoded and thresholded before the soft-NMS")
    ap.add_argument("--device", default="cuda:0", help="the GPU (under torch.distributed.run with NCCL: cuda:LOCAL_RANK)")
    args = ap.parse_args(argv)
    if args.extract_proposals and args.network == "mobilenetv2":
        ap.error("--extract-proposals needs a ResNet-101 network (the MobileNetV2 graph has no RPN-only forward)")
    if args.concurrent_jobs is not None and args.concurrent_jobs < 1:
        ap.error("--concurrent-jobs must be at least 1")
    return args


def config_for(args):
    return IT.default_config(neg=False, autofocus=args.network == "resnet101_autofocus",
                             network="mobilenetv2" if args.network == "mobilenetv2" else "resnet101",
                             dataset="pascal_voc" if args.dataset == "PascalVOC" else "coco")


def load_imdb(args, image_set, world, rank):
    """(imdb, roidb) of one image set: the GT roidb, whose boxes the proposal recall is scored against.  Rank 0 reads
    the annotations first and writes the caches the other ranks then read."""
    def load():
        imdb = load_data.DATASETS[args.dataset](image_set, args.root_path, args.dataset_path,
                                                os.path.dirname(os.path.abspath(args.prefix)), device=args.device)
        return imdb, [dict(r) for r in imdb.gt_roidb()]
    if rank == 0:
        out = load()
    if world > 1:
        torch.distributed.barrier()
        if rank != 0:
            out = load()
    return out


def main(argv=None):
    """Returns dict(world_size, rank, results={image set: (all_boxes or proposals, stats)}); ranks other than 0 hold
    None in place of the boxes.  A process group this call initialised is destroyed before it returns."""
    args = parse_args(argv)
    dist = torch.distributed
    owned = not (dist.is_available() and dist.is_initialized())
    world, rank = init_distributed(args)
    group = dist.group.WORLD if world > 1 else None
    jobs = args.concurrent_jobs or world
    logging.basicConfig(level=logging.INFO if rank == 0 else logging.WARNING, format="%(asctime)s %(message)s")
    log = logging.getLogger()
    try:
        cfg = config_for(args)
        net = load_test_net(args, cfg, args.epoch)
        out = dict(world_size=world, rank=rank, results={})
        for image_set in args.image_set.split('+'):
            imdb, roidb = load_imdb(args, image_set, world, rank)
            cfg.dataset.test_image_set = image_set
            if args.extract_proposals:
                res, stats = tester.imdb_proposal_extraction_wrapper(
                    net, cfg, roidb, args.proposal_save_path, device=args.device, image_loader=host.imread, imdb=imdb,
                    concurrent_jobs=jobs, group=group)
                log.info("%s: proposals of %d images in %s\n%s", image_set, len(roidb),
                         os.path.join(args.proposal_save_path, tester.proposal_file_name(cfg)), stats.get("recall"))
            else:
                res, stats = tester.imdb_detection_wrapper(
                    net, cfg, roidb, num_classes=cfg.dataset.NUM_CLASSES, device=args.device, imdb=imdb,
                    detect_backend=args.detect_backend, image_loader=host.imread, concurrent_jobs=jobs, group=group)
                log.info("%s: detections of %d images\n%s", image_set, len(roidb), stats.get("eval"))
            out["results"][image_set] = (res, stats)
        return out
    finally:
        if owned and world > 1:
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
