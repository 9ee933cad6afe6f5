"""Seeded inputs of the inference proposal operator (ops.multi_proposal) at the geometry the Tester runs, shared by
tests/test_multi_proposal_exact_gpu.py (CUDA path vs oracle/mp_cpuop.c, byte for byte) and
tests/test_multi_proposal_cases_cpu.py (the builders produce what they claim).

Geometry comes from the code: the network's config (iterator.default_config), its TEST.SCALES / BATCH_IMAGES, the
test iterator's resize rule (chips_inference.image_scale) and canvas (tester._canvas_size).  A case holds NCHW arrays
(what the oracle reads) and the layout the device is called with."""
import functools
import inspect
import math

import numpy as np

from sniper_b200 import chips_inference, iterator, tester

NETWORKS = ("resnet101", "mobilenetv2")
# COCO-sized originals (width, height); a batch holds images of one orientation, as MNIteratorTestAutoFocus groups them
LANDSCAPE = ((1333, 800), (640, 427), (500, 375), (200, 150))
PORTRAIT = ((800, 1333), (427, 640), (375, 500), (150, 200))
ONE_BELOW_ONE = np.float32(np.nextafter(np.float32(1.0), np.float32(0.0)))    # 0.99999994f
BIG_DELTA = 8.0       # exp(8) x any anchor: the decoded box covers the whole image, so it clips to the image exactly


@functools.lru_cache(maxsize=None)
def graph(network):
    """The inference graph's proposal parameters: stride, anchor set, pre-NMS count and the padded RPN head width (the
    head conv's output channels are rounded up to a multiple of 32: 128 for ResNet-101's 6 x 21, 96 for MobileNetV2's
    6 x 15; the deltas are channels 0:4A)."""
    from sniper_b200 import model_mnv2, ops
    cfg = iterator.default_config(network=network)
    n = cfg.network
    A = int(n.NUM_ANCHORS)
    assert A == len(n.ANCHOR_SCALES) * len(n.ANCHOR_RATIOS)
    if network == "mobilenetv2":
        pre = inspect.signature(model_mnv2.SniperMobileNetV2.forward_inference).parameters["rpn_pre_nms_top_n"].default
    else:
        pre = inspect.signature(ops.multi_proposal).parameters["rpn_pre_nms_top_n"].default
    return dict(feat_stride=int(n.RPN_FEAT_STRIDE), scales=tuple(n.ANCHOR_SCALES), ratios=tuple(n.ANCHOR_RATIOS), A=A,
                pre=int(pre), head_c=(6 * A + 31) // 32 * 32)


def tester_batch(network, scale_i, sizes, crops=None):
    """One MNIteratorTestAutoFocus batch at TEST.SCALES[scale_i] of whole images (width, height), or of crops (width,
    height) of them (the FocusChips of the later AutoFocus scales; an image's scale is that of the whole image):
    im_info [n,3] = (resized h, resized w, scale) per entry and the feature map (H, W) of the canvas padded to the
    largest entry."""
    cfg = iterator.default_config(network=network)
    stride = int(cfg.network.RPN_FEAT_STRIDE)
    target = cfg.TEST.SCALES[scale_i]
    rows, mh, mw = [], 0, 0
    for k, (w, h) in enumerate(sizes):
        s = chips_inference.image_scale(w, h, target)
        cw, ch = crops[k] if crops is not None else (w, h)
        mh, mw = max(mh, int(math.ceil(ch * s))), max(mw, int(math.ceil(cw * s)))
        rows.append((int(np.rint(ch * s)), int(np.rint(cw * s)), s))
    SH, SW = tester._canvas_size(mh, mw, stride)
    assert SH % stride == 0 and SW % stride == 0
    im_info = np.array([(min(dh, SH), min(dw, SW), s) for dh, dw, s in rows], np.float32)
    return im_info, SH // stride, SW // stride


def batch_sizes(network, scale_i, orientation):
    """BATCH_IMAGES[scale_i] images of one orientation, cycling through the COCO-sized ones and a small one."""
    n = int(iterator.default_config(network=network).TEST.BATCH_IMAGES[scale_i])
    pool = LANDSCAPE if orientation == "landscape" else PORTRAIT
    return [pool[i % len(pool)] for i in range(max(n, 2))]


# ---------------------------------------------------------------------------------------------------- score regimes
def _pairs(fg):
    """(bg, fg) softmax pairs as the RPN's SoftmaxActivation leaves them: cls_prob [B,2A,H,W] from fg [B,A,H,W]."""
    fg = fg.astype(np.float32)
    return np.concatenate([(np.float32(1) - fg), fg], 1)


def _tie_free(rng, shape, lo=0.0, hi=1.0):
    n = int(np.prod(shape))
    v = lo + (hi - lo) * (rng.permutation(n) + 1.0) / (n + 1.0)
    fg = v.astype(np.float32).reshape(shape)
    assert len(np.unique(fg)) == n
    return fg


def strip_pairs(H, W):
    """(anchor type, h, w1, w2) of the pairs the FastNMS overlap map must NOT list on an H x W map with H <= 16 < W:
    anchor type 20 (ratio 2, scale 24 at stride 16, 264 x 528 px) against itself at column offset 16 or 17.  The map
    applies a column offset as a vertical shift, where those anchors still overlap by IoU >= 0.3, but a column offset
    >= H is out of the map's rows (multi_proposal.cu's swapped (row, column) bounds).  The pairs lie 5 rows and 24
    columns apart, too far for the map to list one pair's anchors for another's."""
    assert H <= 16 and W >= 58
    return [(20, h, w1, w1 + 16 + q % 2) for q, (h, w1) in enumerate(zip(range(0, H, 5), (0, 40) * 4))]


def scores(regime, rng, B, A, H, W, pre, inside=None):
    """fg scores [B,A,H,W] of one regime and the per-row delta override (None or a bool mask [B,A,H,W] of rows whose
    deltas become BIG_DELTA, i.e. whole-image boxes).  inside: bool [A*H*W], anchors centred inside every image of the
    batch (their boxes survive the clip and the minimum size)."""
    shape = (B, A, H, W)
    n = A * H * W
    big = None
    if regime == "tie_free":
        fg = _tie_free(rng, shape)
    elif regime == "quantised":
        # logits on a 1/256 grid: the softmax maps each grid difference to one float, so score values repeat in short
        # runs (shorter than a 64-row trip of the bit-mask NMS among its candidates)
        lg = np.round(rng.randn(B, 2, n) * 512.0) / 256.0
        e = np.exp(lg - lg.max(1, keepdims=True))
        fg = (e / e.sum(1, keepdims=True))[:, 1].astype(np.float32).reshape(shape)
    elif regime == "saturated":
        # a trained RPN's saturated softmax: thousands of anchors at exactly 1.0f and at the float below it
        fg = _tie_free(rng, shape, 0.0, 0.999).reshape(B, n)
        m = min(3000, n // 4)
        for b in range(B):
            idx = rng.permutation(n)
            fg[b, idx[:m]] = 1.0
            fg[b, idx[m:2 * m]] = ONE_BELOW_ONE
        fg = fg.reshape(shape)
    elif regime == "k_boundary":
        # rank K of the pre-NMS selection inside one run of equal scores: rows above the run decode to the whole image
        # (one survives the NMS), so the output is decided by which rows of the run the selection took
        assert n > pre + 64
        fg = _tie_free(rng, shape, 0.0, 0.5).reshape(B, n)
        big = np.zeros((B, n), bool)
        for b in range(B):
            idx = rng.permutation(np.flatnonzero(inside))
            top, run = idx[:pre - 40], idx[pre - 40:pre + 60]
            fg[b, top] = _tie_free(rng, (len(top),), 0.6, 1.0)
            fg[b, run] = 0.55
            big[b, top] = True
        fg, big = fg.reshape(shape), big.reshape(shape)
    elif regime == "long_run":
        # 10 distinct top scores, then a run of 100 equal ones: longer than a 64-row trip of the bit-mask NMS
        fg = _tie_free(rng, shape, 0.0, 0.97).reshape(B, n)
        for b in range(B):
            idx = rng.permutation(n)
            fg[b, idx[:10]] = _tie_free(rng, (10,), 0.99, 1.0)
            fg[b, idx[10:110]] = 0.98
        fg = fg.reshape(shape)
    elif regime == "strip_pairs":
        # the top rows are the strip_pairs, all decoding to the whole image: kept both unless the map lists the pair
        fg = _tie_free(rng, shape, 0.0, 0.9)
        big = np.zeros(shape, bool)
        pairs = strip_pairs(H, W)
        for b in range(B):
            top = _tie_free(rng, (2 * len(pairs),), 0.9, 1.0)
            for q, (a, h, w1, w2) in enumerate(pairs):
                fg[b, a, h, w1], fg[b, a, h, w2] = top[2 * q], top[2 * q + 1]
                big[b, a, h, w1] = big[b, a, h, w2] = True
    else:
        raise ValueError(regime)
    return fg, big


def deltas(rng, B, A, H, W, big=None, filler_image=None):
    """bbox_pred [B,4A,H,W]; rows of `big` decode to the whole image; in image `filler_image` all but 150 anchors shrink
    below the 3-pixel minimum size, so fewer than R rows survive and filler rows follow."""
    d = (rng.randn(B, A, 4, H, W) * 0.3).astype(np.float32)
    if big is not None:
        d[:, :, 2][big] = BIG_DELTA
        d[:, :, 3][big] = BIG_DELTA
    if filler_image is not None:
        keep = np.zeros(A * H * W, bool)
        keep[rng.permutation(A * H * W)[:150]] = True
        keep = keep.reshape(A, H, W)
        d[filler_image, :, 2][~keep] = -8.0
        d[filler_image, :, 3][~keep] = -8.0
    return d.reshape(B, 4 * A, H, W)


# ---------------------------------------------------------------------------------------------------- layouts
def device_inputs(cls_prob, bbox_pred, layout, head_c):
    """(cls_prob, bbox_pred) as ops.multi_proposal is called: "nchw"; "nhwc" (contiguous, 2A / 4A channels); "graph"
    (model.rpn_proposals: prob [B,H,W,2A], bbox_pred = the padded head [B,H,W,head_c] with the deltas in channels 0:4A
    and NaN in every other channel, so a read past the deltas shows in the output)."""
    if layout == "nchw":
        return cls_prob, bbox_pred
    prob = np.ascontiguousarray(cls_prob.transpose(0, 2, 3, 1))
    d = np.ascontiguousarray(bbox_pred.transpose(0, 2, 3, 1))
    if layout == "nhwc":
        return prob, d
    assert layout == "graph"
    head = np.full(d.shape[:3] + (head_c,), np.nan, np.float32)
    head[..., :d.shape[3]] = d
    return prob, head


# ---------------------------------------------------------------------------------------------------- cases
def _case(name, network, scale_i, orientation, layout, regime, flags=0, filler=False, seed=0, crops=None):
    return dict(name=name, network=network, scale_i=scale_i, orientation=orientation, layout=layout, regime=regime,
                flags=flags, filler=filler, seed=seed, crops=crops)


# FocusChips of landscape COCO images at the ResNet-101 graph's middle scale: wide strips, a 16 x 80 map
FOCUS_STRIPS = ((600, 120), (640, 130), (380, 96), (520, 110))


def _cases():
    out = []
    layouts = ("graph", "nchw", "nhwc")
    regimes = ("tie_free", "quantised", "saturated")
    k = 0
    for network in NETWORKS:
        for scale_i in range(3):
            for orientation in ("landscape", "portrait"):
                # every Tester canvas of both graphs, one layout and one regime each (rotating), plain flags
                name = "%s-s%d-%s" % (network, scale_i, orientation)
                out.append(_case(name, network, scale_i, orientation, layouts[k % 3], regimes[(k // 2) % 3], seed=k))
                k += 1
    # the largest canvases in the graph's own layout with each tie regime; the flags of the reference's GPU build
    big = {"resnet101": 2, "mobilenetv2": 0}
    for network in NETWORKS:
        s = big[network]
        for regime in ("tie_free", "quantised", "saturated", "long_run", "k_boundary"):
            out.append(_case("%s-largest-%s" % (network, regime), network, s, "landscape", "graph", regime, seed=k))
            k += 1
        out.append(_case("%s-largest-suppress" % network, network, s, "portrait", "graph", "quantised", flags=1, seed=k))
        out.append(_case("%s-largest-fastnms" % network, network, s, "landscape", "graph", "tie_free", flags=2,
                         seed=k + 1))
        out.append(_case("%s-mid-fastnms-suppress" % network, network, 1, "portrait", "nchw", "saturated", flags=3,
                         seed=k + 2))
        out.append(_case("%s-mid-filler" % network, network, 1, "landscape", "nhwc", "quantised", filler=True,
                         seed=k + 3))
        k += 4
    # FastNMS on a map shorter than the largest anchor's reach: the overlap map's swapped (row, column) bounds matter
    for flags in (2, 3):
        out.append(_case("resnet101-focuschips-strip-pairs-flags%d" % flags, "resnet101", 1, "landscape", "graph",
                         "strip_pairs", flags=flags, seed=k, crops=FOCUS_STRIPS))
        k += 1
    # a map below pre_nms (no selection) with every regime that applies there
    for regime in ("saturated", "long_run"):
        out.append(_case("mobilenetv2-small-%s" % regime, "mobilenetv2", 2, "landscape", "graph", regime, seed=k))
        k += 1
    return out


CASES = _cases()
CASE_NAMES = [c["name"] for c in CASES]


@functools.lru_cache(maxsize=None)
def build(name):
    """dict(cls_prob, bbox_pred (NCHW, for the oracle), im_info, kw (ops.multi_proposal geometry), pre, layout, flags,
    H, W, A, graph) of case `name`."""
    c = next(c for c in CASES if c["name"] == name)
    g = graph(c["network"])
    sizes = batch_sizes(c["network"], c["scale_i"], c["orientation"])
    crops = None
    if c["crops"] is not None:
        crops = [c["crops"][i % len(c["crops"])] for i in range(len(sizes))]
        sizes = [(640, 427)] * len(sizes)
    im_info, H, W = tester_batch(c["network"], c["scale_i"], sizes, crops)
    B, A = len(sizes), g["A"]
    rng = np.random.RandomState(7000 + c["seed"])
    stride = g["feat_stride"]
    ctr = (stride - 1) / 2.0
    inside = ((np.arange(H)[:, None] * stride + ctr < im_info[:, 0].min()) &
              (np.arange(W)[None, :] * stride + ctr < im_info[:, 1].min()))
    fg, big = scores(c["regime"], rng, B, A, H, W, g["pre"], np.tile(inside.ravel(), A))
    bbox_pred = deltas(rng, B, A, H, W, big, filler_image=B - 1 if c["filler"] else None)
    kw = dict(feat_stride=g["feat_stride"], scales=g["scales"], ratios=g["ratios"])
    return dict(c, cls_prob=_pairs(fg), bbox_pred=bbox_pred, im_info=im_info, kw=kw, pre=g["pre"], H=H, W=W, A=A,
                head_c=g["head_c"])


def tied_pair(overlap):
    """Two rows with equal top scores on a 16 x 16 ResNet-101 map (5376 anchors: no pre-NMS selection, so the rows are
    the anchor indices).  overlap=False: rows 1 and 32, boxes apart -- both are kept, row 1 first (row 32 is lane 0 of
    warp 1, row 1 lane 1 of warp 0: the training operator's scan order would take 32 first).  overlap=True: rows 5 and
    1026 decode to the same whole-image box -- row 5 must be kept and 1026 suppressed.  Returns (cls_prob, bbox_pred,
    im_info, (i, j))."""
    rng = np.random.RandomState(91 if overlap else 90)
    B, A, H, W = 1, 21, 16, 16
    fg = _tie_free(rng, (B, A * H * W), 0.0, 0.9)
    d = (rng.randn(B, A, 4, H * W) * 0.3).astype(np.float32).reshape(B, A * 4, H * W)
    i, j = (5, 1026) if overlap else (1, 32)
    fg[0, [i, j]] = 0.95
    for r in (i, j):
        a, hw = divmod(r, H * W)
        d[0, 4 * a:4 * a + 4, hw] = (0.0, 0.0, BIG_DELTA, BIG_DELTA) if overlap else 0.0
    im_info = np.array([[H * 16, W * 16, 1.0]], np.float32)
    return _pairs(fg.reshape(B, A, H, W)), d.reshape(B, 4 * A, H, W), im_info, (i, j)
