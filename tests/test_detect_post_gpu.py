"""The device detection backend (`sniper_detect_post`, `inference.DeviceDetections`, `Tester.get_detections(backend=
"device")`) against the host path it mirrors: `inference.detect_postprocess` -> `threshold_detections` -> the valid-range
step of `aggregate`.

The kernel decodes in float64 with the exponential taken in double.  The host functions do the same when they are
given float64 deltas, and that is the strict comparison below (same rows in the same order, scores byte-equal,
coordinates equal up to rare 1-ulp differences of the two double `exp`).  `Tester.detect` hands them the float32 deltas,
on which `np.exp` is numpy's float32 routine (a few float32 ulp from the correctly rounded value on many inputs), so
against that literal call coordinates agree to ~1e-4 px rather than to the last bit; that difference is measured and
bounded separately."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

B, R, K = 8, 300, 81
SIZES = [(640, 480), (420, 610), (512, 512), (333, 500)]                 # (width, height): landscape, portrait, square


def _roidb():
    """Four images; chips whose left / top / right / bottom border is the image border, and interior ones."""
    db = []
    for w, h in SIZES:
        crops = np.array([[0.0, 0.0, w, h],                               # the whole image: no border is tested
                          [0.25, 30.0, w * 0.6, h * 0.7],                 # cx1 < 0.5
                          [w * 0.2, 20.5, w - 0.25, h - 40.0],            # cx2 >= w - 0.5
                          [50.5, 40.25, w * 0.8 + 0.125, h * 0.75]])      # interior
        db.append(dict(width=w, height=h, inference_crops=crops))
    return db


def _inputs(seed, sigma=10.0, B=B, R=R, K=K):
    import torch
    from sniper_b200 import ops, synth
    rng = np.random.RandomState(seed)
    H, W = 32, 40
    cls, bbox = synth.rpn_outputs(rng, B, 21, H, W)
    im_info = np.array([[rng.randint(300, 16 * H + 1), rng.randint(400, 16 * W + 1), s]
                        for s in (0.6, 1.0, 1.6667, 2.5, 0.8, 1.2, 3.0, 0.4375)[:B]], np.float32)
    info = torch.from_numpy(im_info).cuda()
    rois, _ = ops.multi_proposal(torch.from_numpy(cls).cuda(), torch.from_numpy(bbox).cuda(), info, rpn_post_nms_top_n=R)
    z = rng.randn(B * R, K) * sigma
    e = np.exp(z - z.max(1, keepdims=True))
    cls_prob = torch.from_numpy((e / e.sum(1, keepdims=True)).astype(np.float32)).cuda()
    wide = torch.from_numpy((rng.randn(B * R, K + 4 + 3) * 0.5).astype(np.float32)).cuda()
    deltas = wide[:, K:K + 4]                                            # the strided view the R-FCN head returns
    assert not deltas.is_contiguous()
    return rois, cls_prob, deltas, info


def _host_rows(rois, cls_prob, deltas, im_info, db, im_ids, chip_ids, prune, vr, delta_dtype=np.float64, thresh=1e-3):
    """What the host path keeps, as {(image, chip, class): float32 [n,5]} in roi order."""
    from sniper_b200 import inference
    nb, k = im_info.shape[0], cls_prob.shape[1]
    scores, preds = inference.detect_postprocess(rois.cpu().numpy(), cls_prob.cpu().numpy(),
                                                 deltas.cpu().numpy().astype(delta_dtype), im_info.cpu().numpy(), nb)
    out = {}
    for b in range(nb):
        r = db[im_ids[b]]
        pr = (r['inference_crops'][chip_ids[b]], r['width'], r['height']) if prune else None
        dets = inference.threshold_detections(scores[b], preds[b], k, thresh, prune=pr)
        for j in range(1, k):
            d = np.asarray(dets[j], np.float32).reshape(-1, 5)
            areas = (d[:, 3] - d[:, 1]) * (d[:, 2] - d[:, 0])             # inference.aggregate's valid-range step
            keep = np.ones(len(d), bool)
            if vr[0] > 0:
                keep &= areas > vr[0] * vr[0]
            if vr[1] > 0:
                keep &= areas <= vr[1] * vr[1]
            out[(im_ids[b], chip_ids[b], j)] = d[keep]
    return out


def _device_rows(rois, cls_prob, deltas, im_info, db, im_ids, chip_ids, prune, vr, scale=0, dets=None):
    from sniper_b200 import inference
    dets = dets or inference.DeviceDetections("cuda")
    dets.append(rois, cls_prob, deltas, im_info, inference.chip_table(db, im_ids, chip_ids, prune, vr), scale=scale)
    rows, keys = dets.result()
    return rows.cpu().numpy(), keys.cpu().numpy()


def _ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


IM_IDS = [0, 0, 1, 1, 2, 2, 3, 3]
CHIP_IDS = [1, 2, 3, 0, 2, 1, 3, 1]


@pytest.mark.parametrize("prune", [False, True])
@pytest.mark.parametrize("vr", [(40, -1), (16, 90), (-1, 40)])
def test_kernel_keeps_the_rows_of_the_host_path(prune, vr):
    from sniper_b200 import inference
    db = _roidb()
    rois, cls_prob, deltas, info = _inputs(11)
    rows, keys = _device_rows(rois, cls_prob, deltas, info, db, IM_IDS, CHIP_IDS, prune, vr, scale=1)
    order = np.argsort(keys, kind="stable")
    rows, keys = rows[order], keys[order]
    img, cls, scale, chip, roi = inference.unpack_key(keys)
    assert (scale == 1).all() and len(np.unique(keys)) == len(keys)
    want = _host_rows(rois, cls_prob, deltas, info, db, IM_IDS, CHIP_IDS, prune, vr)
    # the sorted run is the host's rows, image by image, class by class, chip by chip, in roi order
    exp = [want[(i, c, j)] for i in range(len(db)) for j in range(1, K)
           for c in sorted(ch for im, ch in zip(IM_IDS, CHIP_IDS) if im == i)]
    exp = np.concatenate(exp, 0)
    passing = float((cls_prob[:, 1:] > 1e-3).float().mean())
    print("passing the threshold: %.2f %% of %d scores; kept %d rows" % (100 * passing, B * R * (K - 1), len(rows)))
    assert 0.01 < passing < 0.2 and len(exp) > 1000
    assert rows.shape == exp.shape
    assert rows[:, 4].tobytes() == exp[:, 4].tobytes()
    # the key names the row: its score is cls_prob[chip's batch slot * R + roi, class]
    slot = {(i, c): b for b, (i, c) in enumerate(zip(IM_IDS, CHIP_IDS))}
    src = np.array([slot[(i, c)] for i, c in zip(img, chip)]) * R + roi
    assert np.array_equal(cls_prob.cpu().numpy()[src, cls], rows[:, 4])
    u = _ulps(rows[:, :4], exp[:, :4]).max(1)
    print("rows off by one float32 ulp: %d of %d" % (int((u > 0).sum()), len(u)))
    assert u.max(initial=0) <= 1 and (u > 0).sum() <= 1e-4 * len(u)


def test_literal_float32_deltas_differ_only_by_the_float32_exp():
    """`Tester.detect` feeds float32 deltas, so numpy takes their exponential in float32.  Without pruning and without
    a valid range the kept set depends on the scores alone: the same rows, coordinates within numpy's float32 exp
    error on the predicted size (<= 3 ulp of a size of at most a few thousand pixels, over a scale >= 0.4)."""
    db = _roidb()
    rois, cls_prob, deltas, info = _inputs(12)
    rows, keys = _device_rows(rois, cls_prob, deltas, info, db, IM_IDS, CHIP_IDS, False, (-1, -1))
    want = _host_rows(rois, cls_prob, deltas, info, db, IM_IDS, CHIP_IDS, False, (-1, -1), delta_dtype=np.float32)
    # both sides into key order: the host's lists come per (slot, class) in roi order
    exp = np.concatenate([want[(i, c, j)] for i, c in zip(IM_IDS, CHIP_IDS) for j in range(1, K)], 0)
    order = np.argsort(keys, kind="stable")
    rows = rows[order]
    exp_keys = []
    p = cls_prob.cpu().numpy()
    for b, (i, c) in enumerate(zip(IM_IDS, CHIP_IDS)):
        for j in range(1, K):
            for r in np.nonzero(p[b * R:(b + 1) * R, j] > np.float32(1e-3))[0]:
                exp_keys.append((i << 44) | (j << 34) | (c << 16) | int(r))
    exp = exp[np.argsort(np.array(exp_keys, np.int64), kind="stable")]
    assert rows.shape == exp.shape and rows[:, 4].tobytes() == exp[:, 4].tobytes()
    d = np.abs(rows[:, :4].astype(np.float64) - exp[:, :4])
    print("float32-exp host path: %d of %d rows differ, max %.3g px, max %d ulp"
          % (int((d.max(1) > 0).sum()), len(d), d.max(), int(_ulps(rows[:, :4], exp[:, :4]).max())))
    assert d.max() < 2e-3


def test_two_launches_are_byte_identical():
    import torch
    db = _roidb()
    rois, cls_prob, deltas, info = _inputs(13)
    runs = []
    for _ in range(2):
        from sniper_b200 import inference
        dets = inference.DeviceDetections("cuda")
        dets.rows.fill_(float("nan"))
        dets.keys.fill_(-1)
        for scale in (0, 1):
            dets.append(rois, cls_prob, deltas, info, inference.chip_table(db, IM_IDS, CHIP_IDS, True, (16, 90)),
                        scale=scale)
        n = len(dets)
        runs.append((n, dets.rows.clone(), dets.keys.clone()))
    assert runs[0][0] == runs[1][0] > 0
    n = runs[0][0]
    assert torch.equal(runs[0][2], runs[1][2])
    assert runs[0][1][:n].cpu().numpy().tobytes() == runs[1][1][:n].cpu().numpy().tobytes()
    assert (runs[0][2][n:] == -1).all()                                  # nothing written past the cursor


def _all_pass(nb=2, r=50, k=81, seed=3):
    """A batch whose every score passes 1e-3: nb * r * (k - 1) rows."""
    import torch
    rng = np.random.RandomState(seed)
    rois = np.zeros((nb * r, 5), np.float32)
    rois[:, 0] = np.repeat(np.arange(nb), r)
    xy = rng.uniform(0, 200, (nb * r, 2))
    rois[:, 1:3], rois[:, 3:5] = xy, xy + rng.uniform(8, 200, (nb * r, 2))
    cls_prob = torch.full((nb * r, k), 1.0 / k) + torch.from_numpy(rng.uniform(0, 1e-4, (nb * r, k))).float()
    deltas = torch.from_numpy((rng.randn(nb * r, 4) * 0.5).astype(np.float32))
    info = torch.tensor([[400.0, 420.0, 1.0]] * nb)
    db = [dict(width=420, height=400, inference_crops=np.array([[0.0, 0.0, 420.0, 400.0]] * nb))]
    return [t.cuda() for t in (torch.from_numpy(rois), cls_prob, deltas, info)], db


def test_chip_without_detections_and_skipped_chip():
    from sniper_b200 import inference
    db = _roidb()
    rois, cls_prob, deltas, info = _inputs(14)
    cls_prob = cls_prob.clone()
    cls_prob[2 * R:3 * R] = 0.0
    cls_prob[2 * R:3 * R, 0] = 1.0                                       # slot 2: background only
    table = inference.chip_table(db, IM_IDS, CHIP_IDS, False, (-1, -1))
    table[5, 0] = -1.0                                                   # slot 5: a repeated chip
    dets = inference.DeviceDetections("cuda")
    dets.append(rois, cls_prob, deltas, info, table)
    rows, keys = dets.result()
    img, _, _, chip, _ = inference.unpack_key(keys.cpu().numpy())
    got = set(zip(img.tolist(), chip.tolist()))
    assert got == {(i, c) for b, (i, c) in enumerate(zip(IM_IDS, CHIP_IDS)) if b not in (2, 5)}
    p = cls_prob.cpu().numpy()
    keep = np.ones(B * R, bool)
    keep[2 * R:3 * R] = keep[5 * R:6 * R] = False
    assert len(rows) == int((p[keep, 1:] > np.float32(1e-3)).sum())


def test_full_buffer_growth_and_refusal():
    import torch
    from sniper_b200 import inference, ops
    from sniper_b200._lib import SniperError
    (rois, cls_prob, deltas, info), db = _all_pass()
    table = inference.chip_table(db, [0, 0], [0, 1], False, (-1, -1))
    worst = rois.shape[0] * (K - 1)
    # every score passes: the batch fills a fixed buffer of exactly B * R * (K - 1) rows
    full = inference.DeviceDetections("cuda", capacity=worst, growable=False)
    full.append(rois, cls_prob, deltas, info, table)
    assert len(full) == worst == full.capacity
    assert torch.isfinite(full.rows).all() and len(torch.unique(full.keys)) == worst
    # ... and cannot take a second batch: refused on the host, before any launch, with nothing touched
    before = (full.rows.clone(), full.keys.clone())
    with pytest.raises(SniperError, match="run buffer of %d rows cannot take this batch" % worst):
        full.append(rois, cls_prob, deltas, info, table, scale=1)
    assert len(full) == worst and torch.equal(full.rows, before[0]) and torch.equal(full.keys, before[1])
    small = inference.DeviceDetections("cuda", capacity=worst - 1, growable=False)
    with pytest.raises(SniperError, match="cannot take this batch"):
        small.append(rois, cls_prob, deltas, info, table)
    assert len(small) == 0
    # a caller that understates its bound: the launch finds the rows not fitting, writes none and says how many it needed
    ops.detect_post(rois, cls_prob, deltas, info, torch.from_numpy(table).cuda(), full.rows, full.keys, full.state,
                    full.workspace, scale=1, rows_bound=0)
    assert full.state.cpu().tolist() == [worst, 2 * worst]
    assert torch.equal(full.rows, before[0]) and torch.equal(full.keys, before[1])
    full._n = None
    with pytest.raises(SniperError, match="needed %d rows" % (2 * worst)):
        full.finish()
    # a growable buffer that starts at one batch takes three, and holds what a large one holds
    grow = inference.DeviceDetections("cuda", capacity=worst)
    big = inference.DeviceDetections("cuda", capacity=4 * worst, growable=False)
    for scale in range(3):
        for d in (grow, big):
            d.append(rois, cls_prob, deltas, info, table, scale=scale)
    assert len(grow) == len(big) == 3 * worst and grow.capacity >= 3 * worst > worst
    (r0, k0), (r1, k1) = grow.result(), big.result()
    assert torch.equal(k0, k1) and r0.cpu().numpy().tobytes() == r1.cpu().numpy().tobytes()


def _small_cfg():
    from sniper_b200 import iterator as IT
    cfg = IT.default_config()
    cfg.TEST.SCALES = [(96, 160), (192, 320), (288, 480)]
    cfg.TEST.BATCH_IMAGES = [2, 2, 1]
    cfg.TEST.VALID_RANGES = [(40, -1), (16, 90), (-1, 40)]
    cfg.TEST.CHIP_HYPERPARAMS = [(3, 0.3, 4), (3, 0.4, 5)]
    return cfg


def test_pyramid_with_device_detections_equals_host_detections():
    """The fixture of test_autofocus_pyramid_runs_and_device_nms_equals_host_nms.  The host backend decodes with numpy's
    float32 exp (see the module docstring), so boxes are compared to 1e-3 px and scores to 1e-5, not to the last bit."""
    import torch
    from sniper_b200 import model, synth_batch
    from sniper_b200 import tester as TS
    cfg = _small_cfg()
    rng = np.random.RandomState(2)
    db = [dict(width=W, height=H, image_data=rng.randint(0, 256, (H, W, 3)).astype(np.uint8))
          for (W, H) in ((320, 240), (240, 320), (300, 200))]
    mc = model.Cfg()
    mc.batch_images = 2
    net = model.SniperResNet101(mc, deform_offset_std=0.01)
    net.train_step(synth_batch.make_batch(2, seed=7, device="cuda"), lr=0.001)
    net.enable_autofocus(seed=3)
    w0 = net.P.w.clone()
    boxes_h, stats_h = TS.imdb_detection_wrapper(net, cfg, db, detect_backend="host")
    chips_h = [np.array(r['inference_crops'], copy=True) for r in db]
    boxes_d, stats_d = TS.imdb_detection_wrapper(net, cfg, db, detect_backend="device")
    for r, c in zip(db, chips_h):
        assert np.array_equal(np.asarray(r['inference_crops']), c)
    assert [s['chips'] for s in stats_d['scales']] == [s['chips'] for s in stats_h['scales']]
    pre = [s['detections_pre_nms'] for s in stats_d['scales']]
    print("detections before the NMS per scale:", pre)
    assert len(pre) == 3 and pre[0] > 0 and all('detections_pre_nms' not in s for s in stats_h['scales'])
    n, worst_box, worst_score = 0, 0.0, 0.0
    for j in range(1, 81):
        for i in range(3):
            a, b = boxes_d[j][i], boxes_h[j][i]
            assert a.shape == b.shape and a.dtype == b.dtype == np.float32
            if len(a):
                worst_box = max(worst_box, float(np.abs(a[:, :4].astype(np.float64) - b[:, :4]).max()))
                worst_score = max(worst_score, float(np.abs(a[:, 4].astype(np.float64) - b[:, 4]).max()))
            n += len(a)
    print("%d final detections; device vs host backend: boxes within %.3g px, scores within %.3g" % (n, worst_box, worst_score))
    assert n > 0 and worst_box < 1e-3 and worst_score < 1e-5
    assert torch.equal(w0, net.P.w)


def test_mobilenet_inference_feeds_the_kernel_unchanged():
    """SniperMobileNetV2.forward_inference (K = 81, stride 32, 300 rois per chip) -> ops.detect_post on its tensors."""
    import torch
    from sniper_b200 import inference, model_mnv2, synth_batch
    mcfg = model_mnv2.MCfg()
    mcfg.batch_images = 2
    mcfg.bf16 = True
    net = model_mnv2.SniperMobileNetV2(mcfg, device="cuda", seed=2)
    batch = synth_batch.make_batch(2, seed=4, device="cuda", A=mcfg.num_anchors, stride=mcfg.feat_stride)
    net.train_step(batch, lr=0.001)
    rois, _, cls_prob, deltas = net.forward_inference(batch["data"], batch["im_info"])
    torch.cuda.synchronize()
    assert cls_prob.shape == (600, 81) and not deltas.is_contiguous()
    db = [dict(width=512, height=512, inference_crops=np.array([[0.0, 0.0, 512.0, 512.0], [100.0, 60.5, 400.0, 380.0]]))]
    thresh = float(np.median(cls_prob[:, 1:].cpu().numpy()))              # random weights: take about half the scores
    for prune, vr in ((False, (-1, -1)), (True, (16, 200))):
        dets = inference.DeviceDetections("cuda")
        dets.append(rois, cls_prob, deltas, batch["im_info"], inference.chip_table(db, [0, 0], [0, 1], prune, vr),
                    cls_thresh=thresh)
        rows, keys = (t.cpu().numpy() for t in dets.result())
        order = np.argsort(keys, kind="stable")
        want = _host_rows(rois, cls_prob, deltas, batch["im_info"], db, [0, 0], [0, 1], prune, vr, thresh=thresh)
        exp = np.concatenate([want[(0, c, j)] for j in range(1, 81) for c in (0, 1)], 0)
        assert rows.shape == exp.shape and len(exp) > 100
        assert rows[order, 4].tobytes() == exp[:, 4].tobytes()
        u = _ulps(rows[order, :4], exp[:, :4])
        assert u.max() <= 1 and (u.max(1) > 0).sum() <= max(1, 1e-4 * len(u))
