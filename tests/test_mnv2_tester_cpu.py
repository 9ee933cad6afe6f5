"""MobileNetV2 detector evaluation on the host: the canvas geometry per backbone stride, the MobileNetV2 TEST block of
`iterator.default_config`, `Tester.detect` / `get_detections(backend="host")` on `SniperMobileNetV2` (float64 fake ops)
against oracle/torch_graph_mnv2.forward_test followed by the reference's post-processing (lib/inference.py:100-139,
291-301), and the checkpoint round trip main_test.py goes through (`*_test` box-regression tensors)."""
import os
import sys

import numpy as np
import pytest
import torch

from sniper_b200 import iterator as IT
from sniper_b200 import tester as TS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
REF = "/root/reference"


@pytest.mark.parametrize("stride, hor, ver", [(16, (800, 1152), (1088, 896)), (32, (800, 1280), (1088, 1024))])
def test_canvas_follows_the_feature_stride(stride, hor, ver):
    """A 640x480 and a 480x640 image at the (800, 1280) test scale: 800 x 1067 and 1067 x 800 pixels, on a canvas whose
    height is a multiple of 32 and width a multiple of 8 * stride, so every layer's output width is a multiple of 8."""
    cfg = IT.default_config(network={16: "resnet101", 32: "mobilenetv2"}[stride])
    assert cfg.network.RPN_FEAT_STRIDE == stride
    rng = np.random.RandomState(0)
    db = [dict(width=W, height=H, image_data=rng.randint(0, 256, (H, W, 3)).astype(np.uint8),
               inference_crops=np.array([[0, 0, W, H]])) for W, H in ((640, 480), (480, 640))]
    canv = [b['canvas'] for b in TS.MNIteratorTestAutoFocus(db, cfg, (800, 1280), batch_size=1, device="cpu")]
    assert canv == [hor, ver]
    canv = [b['canvas'] for b in TS.MNIteratorTest(db, cfg, (800, 1280), batch_size=1, device="cpu")]
    assert canv == [(800, 1280), (1280, 896 if stride == 16 else 1024)]
    for SH, SW in canv + [hor, ver]:
        assert SH % 32 == 0 and SW % (8 * stride) == 0
        for s in (2, 4, 8, 16, 32)[:{16: 4, 32: 5}[stride]]:
            assert (SW // s) % 8 == 0 and SW % s == 0 and SH % s == 0
    for h, w in ((1, 1), (480, 512), (1400, 2000), (1216, 2000)):
        SH, SW = TS._canvas_size(h, w, stride)
        assert SH - 32 < h <= SH and SW - 8 * stride < w <= SW


def test_resnet_canvases_are_unchanged():
    """The stride-16 rule of the ResNet-101 pyramid: width a multiple of 128, as before the stride became a parameter."""
    for h in range(1, 700, 7):
        for w in range(1, 1500, 13):
            assert TS._canvas_size(h, w) == TS._canvas_size(h, w, 16) == (-(-h // 32) * 32, -(-w // 128) * 128)
    cfg = IT.default_config()
    rng = np.random.RandomState(1)
    db = [dict(width=300, height=200, image_data=rng.randint(0, 256, (200, 300, 3)).astype(np.uint8),
               inference_crops=np.array([[0, 0, 300, 200]]))]
    assert next(TS.MNIteratorTestAutoFocus(db, cfg, (160, 256), batch_size=1, device="cpu"))['canvas'] == (160, 256)


# configs/faster/sniper_mobilenetv2_e2e.yml TEST (:179-256) over configs/faster/default_configs.py
_YML_TEST = dict(SCALES=[(1400, 2000), (800, 1280), (480, 512)], BATCH_IMAGES=[2, 2, 4], MAX_PER_IMAGE=200,
                 VALID_RANGES=[(-1, 90), (32, 180), (75, -1)], NMS=-1, NMS_SIGMA=0.55, AUTO_FOCUS=False,
                 DO_PRUNING=[False, False, False], RPN_PRE_NMS_TOP_N=6000, RPN_POST_NMS_TOP_N=300)


def test_mobilenetv2_test_block():
    import inspect
    from sniper_b200 import model_mnv2 as MM
    t = IT.default_config(network="mobilenetv2").TEST
    for k, v in _YML_TEST.items():
        got = getattr(t, k)
        assert (list(map(tuple, got)) if k in ("SCALES", "VALID_RANGES") else got) == v, k
    assert len(t.SCALES) == len(t.BATCH_IMAGES) == len(t.VALID_RANGES) == len(t.DO_PRUNING)
    # what reaches MultiProposal in SniperMobileNetV2.forward_inference
    pre = inspect.signature(MM.SniperMobileNetV2.forward_inference).parameters["rpn_pre_nms_top_n"].default
    assert (pre, MM.MCfg.rpn_post_nms_top_n) == (t.RPN_PRE_NMS_TOP_N, t.RPN_POST_NMS_TOP_N)
    # the ResNet-101 block is the AutoFocus one, untouched
    r = IT.default_config().TEST
    assert r.SCALES == [(480, 512), (800, 1280), (1400, 2000)] and r.BATCH_IMAGES == [8, 8, 2] and r.AUTO_FOCUS
    assert r.VALID_RANGES == [(75, -1), (32, 180), (-1, 75)] and r.NMS == 0.45 and r.DO_PRUNING == [False, True, True]


@pytest.mark.skipif(not os.path.isdir(REF), reason="reference tree not present")
def test_mobilenetv2_test_block_equals_the_reference_yml():
    import run_ref_symbols as R
    ref = R.load_config("sniper_mobilenetv2_e2e.yml").TEST
    t = IT.default_config(network="mobilenetv2").TEST
    for k in _YML_TEST:
        a, b = getattr(t, k), getattr(ref, k)
        if k in ("SCALES", "VALID_RANGES"):
            a, b = [tuple(x) for x in a], [tuple(x) for x in b]
        assert a == b, (k, a, b)
    assert [tuple(x) for x in t.CHIP_HYPERPARAMS] == [tuple(x) for x in ref.CHIP_HYPERPARAMS]


@pytest.fixture
def f64():
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(old)


def _net(monkeypatch, seed=3):
    import fake_ops
    from sniper_b200 import model_mnv2 as MM
    from sniper_b200 import ops
    fake_ops.install(monkeypatch, ops)
    cfg = MM.MCfg()
    cfg.batch_images, cfg.bf16, cfg.wgrad_stream = 2, False, False
    net = MM.SniperMobileNetV2(cfg, device="cpu", seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for bn in net.all_bns():                # non-trivial affine parameters and moving statistics on the real channels
        bn.st.gamma[:bn.C] = torch.empty(bn.C).uniform_(0.8, 1.2, generator=g)
        bn.st.beta[:bn.C] = torch.empty(bn.C).normal_(0, 0.1, generator=g)
        bn.st.moving_mean[:bn.C] = torch.empty(bn.C).normal_(0, 0.2, generator=g)
        bn.st.moving_var[:bn.C] = torch.empty(bn.C).uniform_(0.5, 2.0, generator=g)
    # a wider box regression than N(0, 0.01) gives, so that decoding, clipping and rescaling all matter
    k = net.cfg.num_classes
    net.fc_out.master[k:k + 4] *= 20.0
    net.fc_out.b[k:k + 4] = torch.tensor([0.05, -0.05, 0.1, -0.1])
    return cfg, net


def _reference_detections(rois, cls_prob, deltas, im_info, scales, num_classes, thresh):
    """lib/inference.py Tester.detect (:119-131) + get_detections (:291-301) in float64: per chip and class j >= 1 the
    rows (x1, y1, x2, y2, score) with score > thresh; every class takes its box from columns 0:4 of the 4-wide
    class-agnostic prediction."""
    out = []
    for idx in range(len(scales)):
        cids = np.where(rois[:, 0] == idx)[0]
        b = rois[cids, 1:].astype(np.float64)
        d = deltas[cids].astype(np.float64)
        w, h = b[:, 2] - b[:, 0] + 1.0, b[:, 3] - b[:, 1] + 1.0
        cx, cy = b[:, 0] + 0.5 * (w - 1.0), b[:, 1] + 0.5 * (h - 1.0)
        pcx, pcy = d[:, 0] * w + cx, d[:, 1] * h + cy
        pw, ph = np.exp(d[:, 2]) * w, np.exp(d[:, 3]) * h
        box = np.stack([pcx - 0.5 * (pw - 1.0), pcy - 0.5 * (ph - 1.0), pcx + 0.5 * (pw - 1.0), pcy + 0.5 * (ph - 1.0)], 1)
        box[:, 0::2] = np.maximum(np.minimum(box[:, 0::2], im_info[idx, 1] - 1), 0)
        box[:, 1::2] = np.maximum(np.minimum(box[:, 1::2], im_info[idx, 0] - 1), 0)
        box = box / scales[idx]
        sc = cls_prob[cids]
        per_class = [None]
        for j in range(1, num_classes):
            inds = np.where(sc[:, j] > thresh)[0]
            per_class.append(np.hstack((box[inds, 0:4], sc[inds, j, np.newaxis])))
        out.append(per_class)
    return out


def test_tester_detections_match_the_oracle_and_the_reference_postprocessing(monkeypatch, f64):
    """Tester.detect / get_detections(backend="host") on a SniperMobileNetV2 at a non-square stride-32 canvas
    (2 x 3 x 224 x 512, two chips of different sizes) against forward_test on the same parameters, decoded the way the
    reference decodes them."""
    import oracle_lib as O
    import torch_graph as TG
    import torch_graph_mnv2 as TM
    cfg, net = _net(monkeypatch)
    B, SH, SW, K = 2, 224, 512, cfg.num_classes
    assert TS._canvas_size(SH, SW, 32) == (SH, SW)
    g = torch.Generator().manual_seed(11)
    data = torch.randn(B, 3, SH, SW, generator=g) * 60.0
    im_info = torch.tensor([[224.0, 500.0, 1.25], [180.0, 512.0, 0.8]])
    data[1, :, 180:, :] = 0.0                                    # the padding of the smaller chip
    roidb = [dict(width=400, height=179, inference_crops=np.array([[0, 0, 400, 179]])),
             dict(width=640, height=225, inference_crops=np.array([[0, 0, 640, 225]]))]
    batch = dict(data=data, im_info=im_info, im_ids=np.array([0, 1]), chip_ids=np.array([0, 0]))
    tcfg = IT.default_config(network="mobilenetv2")
    w0 = net.P.w.clone()
    tester = TS.Tester(net, None, roidb, [batch], tcfg, num_classes=K)
    scores, boxes, _, im_ids, maps, chip_ids = tester.detect(batch)
    assert maps == [] and list(im_ids) == [0, 1] and len(scores) == len(boxes) == B
    thresh = 0.0125                                              # about half of the near-uniform random-weight scores
    all_boxes, all_maps = tester.get_detections(cls_thresh=thresh, backend="host")
    assert torch.equal(net.P.w, w0)

    arg, aux = net.export_reference()
    P, Aux = TM.params_to_torch(arg, aux)
    TG.MODE[0] = "exact"

    def proposals(prob, bbox):
        return O.multi_proposal(prob.numpy(), bbox.numpy(), im_info.numpy(), feat_stride=32, scales=cfg.scales,
                                ratios=cfg.ratios, pre=6000, post=300)["rois"]
    ref = TM.forward_test(P, Aux, data, proposals)
    rois = net.forward_inference(data, im_info)[0].numpy().astype(np.float32)
    assert rois.shape == (B * 300, 5) and np.array_equal(rois, ref["rois"])
    info = im_info.numpy().astype(np.float64)
    want = _reference_detections(ref["rois"], ref["cls_prob"].numpy(), ref["bbox_pred"].numpy(), info,
                                 info[:, 2].astype(np.float32), K, thresh)
    n, worst_box, worst_score = 0, 0.0, 0.0
    for i in range(B):
        assert scores[i].shape == (300, K) and boxes[i].shape == (300, 4)
        for j in range(1, K):
            a, b = all_boxes[j][i][0], want[i][j]
            assert a.shape == b.shape, (i, j, a.shape, b.shape)
            if len(a):
                worst_box = max(worst_box, float((np.abs(a[:, :4] - b[:, :4]) / np.maximum(np.abs(b[:, :4]), 1.0)).max()))
                worst_score = max(worst_score, float(np.abs(a[:, 4] - b[:, 4]).max()))
            n += len(a)
        # boxes lie inside the image (the chip is the whole image; clipped to the resized chip, then rescaled)
        rows = np.concatenate([all_boxes[j][i][0] for j in range(1, K)], 0)
        assert (rows[:, :4] >= 0).all() and (rows[:, [0, 2]] <= roidb[i]['width']).all() \
            and (rows[:, [1, 3]] <= roidb[i]['height']).all()
    print("%d detections; against the oracle + reference post-processing: boxes within %.3g (relative), scores "
          "within %.3g" % (n, worst_box, worst_score))
    assert n > 1000 and worst_box < 1e-7 and worst_score < 1e-7


def test_checkpoint_round_trip_gives_the_processed_bbox_pred(monkeypatch, tmp_path):
    """save_checkpoint writes bbox_pred_*_test = bbox_pred_* scaled by the target stds; load_param(process=True) puts them
    over bbox_pred_*; load_reference then gives a net whose export is exactly the processed arrays."""
    from sniper_b200 import checkpoint
    _, net = _net(monkeypatch, seed=3)
    arg, aux = net.export_reference()
    assert arg["bbox_pred_weight"].shape == (4, 512) and arg["bbox_pred_bias"].shape == (4,)
    prefix = str(tmp_path / "mnv2")
    checkpoint.save_checkpoint(prefix, 7, arg, aux)
    parg, paux = checkpoint.load_param(prefix, 7, process=True)
    assert not any(k.endswith("_test") for k in parg) and set(parg) == set(arg)
    stds = np.array(checkpoint.BBOX_STDS_TEST, np.float32)
    assert np.array_equal(parg["bbox_pred_weight"], arg["bbox_pred_weight"] * stds[:, None])
    assert np.array_equal(parg["bbox_pred_bias"], arg["bbox_pred_bias"] * stds)
    _, fresh = _net(monkeypatch, seed=8)
    fresh.load_reference(parg, paux)
    garg, gaux = fresh.export_reference()
    assert set(garg) == set(parg) and set(gaux) == set(paux)
    for k in parg:
        assert garg[k].dtype == parg[k].dtype and garg[k].tobytes() == parg[k].tobytes(), k
    for k in paux:
        assert gaux[k].tobytes() == paux[k].tobytes(), k
