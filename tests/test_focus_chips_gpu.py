"""AutoFocus FocusChips on the device (`sniper_focus_chips`, `ops.focus_chips`, `add_chips` with a `DeviceFocusMaps`)
against the host code they restate, `chips_inference.gmask` / `add_chips`: same chips, same order, byte for byte."""
import math
from types import SimpleNamespace

import numpy as np
import pytest

from sniper_b200 import chips_inference as CI

pytestmark = pytest.mark.gpu


def _passes(fmap, d, thr, ms, imw, imh):
    """How many times gmask's merge loop runs on this map (its loop, counted)."""
    mask = np.array(fmap, copy=True)
    iw, ih = int(math.ceil(float(imw) / 16)), int(math.ceil(float(imh) / 16))
    hi = mask >= thr
    mask[hi] = 1
    mask[~hi] = 0
    mask = CI.dilate(mask, d) * 255
    rects = CI.contour_rects(mask.astype(np.uint8))
    chips, nchips, k = [], -1, 0
    while nchips != len(chips):
        k += 1
        nchips = len(chips)
        for r in rects:
            x, y, w, h = CI._place(*r, ms, iw, ih)
            mask[y:y + h, x:x + w] = 255
        rects = CI.contour_rects(mask.astype(np.uint8))
        chips = rects
    return k


def _run(cases, d, thr, ms):
    """cases: (map float32 [H, W], im_width, im_height, cscale, origin x, origin y).  The maps go to the device as the
    `focus_map` layout does them: channel 1 of a [n, Hmax, Wmax, 2] tensor, read through the strided view.  Returns the
    device chips and the host chips of each case (gmask, then add_chips' shift by the crop origin)."""
    import torch
    from sniper_b200 import ops
    Hm = max(max(c[0].shape[0] for c in cases), 1)
    Wm = max(max(c[0].shape[1] for c in cases), 1)
    full = np.zeros((len(cases), Hm, Wm, 2), np.float32)
    index = np.zeros((len(cases), 6), np.int64)
    geometry = np.zeros((len(cases), 5))
    for m, (fmap, imw, imh, cs, ox, oy) in enumerate(cases):
        H, W = fmap.shape
        full[m, :H, :W, 1] = fmap
        full[m, :H, :W, 0] = 1 - fmap
        index[m] = [0, m, H, W, int(math.ceil(float(imw) / 16)), int(math.ceil(float(imh) / 16))]
        geometry[m] = [imw, imh, cs, ox, oy]
    view = torch.from_numpy(full).cuda()[..., 1]
    assert view.stride(2) == 2
    chips, off = ops.focus_chips([view], index, geometry, d=d, thresh=thr, ms=ms)
    for m, (fmap, imw, imh, cs, ox, oy) in enumerate(cases):
        host = CI.gmask(fmap, d, thr, ms=ms, im_width=imw, im_height=imh, cscale=cs)
        for c in host:
            c[0] += ox
            c[1] += oy
            c[2] += ox
            c[3] += oy
        yield chips[off[m]:off[m + 1]], np.array(host, np.float64).reshape(-1, 4)


def _check(cases, d, thr, ms):
    n = 0
    for m, (dev, host) in enumerate(_run(cases, d, thr, ms)):
        assert dev.shape == host.shape and dev.tobytes() == host.tobytes(), (m, dev, host)
        n += len(host)
    return n


def _case(fmap, imw=None, imh=None, cs=1.0, ox=0.0, oy=0.0):
    H, W = fmap.shape
    return (np.asarray(fmap, np.float32), W * 16.0 if imw is None else imw, H * 16.0 if imh is None else imh, cs, ox, oy)


def test_maps_of_the_host_tests():
    m = np.zeros((32, 40), np.float32)
    m[10, 20] = 0.9
    assert _check([_case(m, 40 * 16, 32 * 16, 2.0)], 3, 0.5, 8) == 1
    m = np.zeros((20, 20), np.float32)
    m[0, 0] = 1.0
    m[19, 19] = 1.0
    assert _check([_case(m, 20 * 16 - 5, 20 * 16)], 3, 0.5, 6) == 2
    rng = np.random.RandomState(3)
    for _ in range(20):
        H, W = rng.randint(12, 40), rng.randint(12, 50)
        m = rng.rand(H, W).astype(np.float32) ** 6
        ms, d = int(rng.choice([4, 8, 16])), int(rng.choice([1, 3, 5]))
        _check([_case(m, W * 16 - int(rng.randint(0, 16)), H * 16 - int(rng.randint(0, 16)))], d, 0.3, ms)


def _right_of_iw(pattern, left=12):
    """The pattern at the right of a map whose iw is `left`: the placed chips of its contours are pushed left of it, so
    the painting never covers the pattern and its contours (holes included) reach the final chips."""
    H, W = pattern.shape
    m = np.zeros((H, left + 2 + W), np.float32)
    m[:, left + 2:] = pattern
    return [_case(m, left * 16.0, H * 16.0, cs=1.5, ox=2.0, oy=1.0), _case(pattern)]


def test_nested_holes_and_connectivity():
    # a ring with a hole holding a ring with a hole holding a blob: four contours
    m = np.zeros((16, 16), np.float32)
    m[1:15, 1:15] = 1
    m[3:13, 3:13] = 0
    m[5:11, 5:11] = 1
    m[7:9, 7:9] = 0
    m[7, 7] = 1
    assert len(CI.contour_rects((m * 255).astype(np.uint8))) == 4
    assert _check(_right_of_iw(m), 1, 0.5, 2) >= 4
    # foreground touching only diagonally: one 8-connected component
    diag = np.eye(9, dtype=np.float32)[:, ::-1]
    assert len(CI.contour_rects((diag * 255).astype(np.uint8))) == 1
    assert _check(_right_of_iw(diag), 1, 0.5, 1) >= 2
    # background reaching the frame only diagonally: still a hole (4-connected background)
    m = np.ones((5, 6), np.float32)
    m[1:4, 1:4] = 0
    m[0, 0] = 0
    m[4, 5] = 0
    m[3, 4] = 0
    assert len(CI.contour_rects((m * 255).astype(np.uint8))) == 2
    assert _check(_right_of_iw(m), 1, 0.5, 1) >= 2
    checker = (np.indices((11, 13)).sum(0) % 2).astype(np.float32)       # every background cell its own 4-region
    assert _check(_right_of_iw(checker, 4), 1, 0.5, 1) >= 1


@pytest.mark.parametrize("d", [1, 2, 3, 4, 5])
def test_every_dilation_size(d):
    rng = np.random.RandomState(d)
    cases = [_case((rng.rand(rng.randint(1, 30), rng.randint(1, 30)) > 0.93).astype(np.float32),
                   cs=float(rng.uniform(0.5, 3))) for _ in range(60)]
    assert _check(cases, d, 0.5, 3) > 0


def test_extents_iw_ih_against_the_map():
    rng = np.random.RandomState(7)
    cases = []
    for dw in (-40, -17, -16, -1, 0, 1, 15, 16, 33):
        for dh in (-20, 0, 9, 31):
            m = (rng.rand(14, 18) > 0.9).astype(np.float32)
            cases.append(_case(m, 18 * 16 + dw, 14 * 16 + dh, cs=1.25, ox=3.5, oy=7.0))
    assert _check(cases, 3, 0.5, 6) > 0
    assert _check(cases, 1, 0.5, 30) > 0                                 # ms larger than the map


def test_threshold_compares_in_float32():
    m = np.full((6, 8), 0.01, np.float32)
    m[2, 3] = np.float32(0.02)                                          # >= 0.02 in float32, < 0.02 in double
    assert m[2, 3] >= 0.02 and float(m[2, 3]) < 0.02
    assert _check([_case(m)], 1, 0.02, 2) == 1
    assert _check([_case(m)], 1, np.float64(0.02), 2) == 0              # numpy compares a float64 scalar in double
    assert _check([_case(m)], 1, 0.0200001, 2) == 0


def test_merge_loop_with_several_passes():
    rng = np.random.RandomState(0)
    cases, most = [], 0
    for _ in range(60):
        H, W = rng.randint(6, 30), rng.randint(6, 30)
        m = (rng.rand(H, W) > 0.9).astype(np.float32)
        cases.append(_case(m))
        most = max(most, _passes(m, 1, 0.5, 3, W * 16, H * 16))
    assert most >= 3
    _check(cases, 1, 0.5, 3)


def test_full_empty_and_thin_maps():
    cases = [_case(np.ones((9, 12))), _case(np.zeros((9, 12))), _case(np.ones((1, 1))), _case(np.zeros((1, 1))),
             _case(np.array([[1, 0, 0, 1, 1, 0, 1]])), _case(np.array([[1, 0, 0, 1, 1, 0, 1]]).T),
             _case(np.array([[0, 1, 0]]))]
    for ms in (1, 2, 5):
        for d in (1, 2, 3):
            _check(cases, d, 0.5, ms)


def test_seeded_random_maps():
    rng = np.random.RandomState(11)
    total = 0
    for rnd in range(6):
        d, ms = int(rng.randint(1, 6)), int(rng.choice([1, 2, 4, 8, 16, 20]))
        thr = float(rng.choice([0.02, 0.2, 0.5]))
        cases = []
        for _ in range(500):
            H, W = int(rng.randint(1, 131)), int(rng.randint(1, 131))
            if rng.rand() < 0.6:
                H, W = min(H, 40), min(W, 40)
            p = float(rng.choice([1, 4, 12, 40]))
            m = (rng.rand(H, W) ** p).astype(np.float32)
            cases.append(_case(m, W * 16 + int(rng.randint(-20, 20)), H * 16 + int(rng.randint(-20, 20)),
                               cs=float(rng.uniform(0.3, 3.0)), ox=float(rng.uniform(0, 900)),
                               oy=float(rng.randint(0, 600))))
        total += _check(cases, d, thr, ms)
    assert total > 1000


def test_large_maps_take_the_workspace():
    """Maps whose scratch does not fit in shared memory (88 x 125 is the largest at a (1400, 2000) scale) run from
    the workspace, mixed with small ones in the same launch; maps with many chips overflow the first launch's room."""
    rng = np.random.RandomState(5)
    cases = [_case((rng.rand(88, 125) > 0.995).astype(np.float32), cs=0.7, ox=10.0),
             _case((rng.rand(130, 130) > 0.999).astype(np.float32)), _case(np.zeros((125, 88))),
             _case((rng.rand(20, 30) > 0.95).astype(np.float32)),
             _case((np.indices((120, 90)).sum(0) % 2).astype(np.float32)),
             _case((rng.rand(100, 110) > 0.7).astype(np.float32))]
    assert _check(cases, 1, 0.5, 1) > 8
    assert _check(cases, 3, 0.5, 4) > 0


def _cfg():
    return SimpleNamespace(TEST=SimpleNamespace(SCALES=[(480, 512), (800, 1280), (1400, 2000)],
                                                CHIP_HYPERPARAMS=[(3, 0.02, 16), (3, 0.2, 20)]))


def _device_maps(roidb, scale, rng, stride=16, batch=3):
    """A DeviceFocusMaps over sparse seeded maps, as the Tester fills it (batches of crops in the iterator's style, a
    crop repeated in a later batch to fill it), and the same maps as host lists."""
    import torch
    crops = [(i, j) for i, r in enumerate(roidb) for j in range(len(r['inference_crops']))]
    crops += crops[:(-len(crops)) % batch]
    maps = CI.DeviceFocusMaps([len(r['inference_crops']) for r in roidb], stride)
    for b0 in range(0, len(crops), batch):
        part = crops[b0:b0 + batch]
        info = np.zeros((len(part), 3), np.float32)
        for k, (i, j) in enumerate(part):
            r, c = roidb[i], roidb[i]['inference_crops'][j]
            s = CI.image_scale(r['width'], r['height'], scale)
            info[k] = [int(np.rint((c[3] - c[1]) * s)), int(np.rint((c[2] - c[0]) * s)), s]
        Hc, Wc = int(math.ceil(info[:, 0].max() / stride)), int(math.ceil(info[:, 1].max() / stride))
        z = torch.from_numpy(rng.randn(len(part), Hc, Wc, 2).astype(np.float32) * 3).cuda()
        z[..., 0] += 12                                                 # sparse FocusPixels at both thresholds
        fm = torch.softmax(z, dim=-1)[..., 1]
        maps.add(fm, info, [i for i, _ in part], [j for _, j in part])
    host = [[maps[i][j] for j in range(len(maps[i]))] for i in range(len(maps))]
    return maps, host


def test_add_chips_on_multi_image_multi_crop_roidbs():
    rng = np.random.RandomState(21)
    cfg = _cfg()
    sizes = [(640, 480), (480, 640), (1333, 800), (500, 375), (800, 1333), (333, 500)]
    db = [dict(width=w, height=h, inference_crops=np.array([[0, 0, w, h]])) for w, h in sizes[:2]]
    db += [dict(width=w, height=h, inference_crops=np.array([[0.0, 0.0, w, h], [w * 0.1, h * 0.2, w * 0.6, h * 0.9],
                                                             [w * 0.45, 12.5, w - 0.5, h * 0.5]])) for w, h in sizes[2:]]
    dbh = [dict(r) for r in db]
    for scale_id in (0, 1):
        maps, host = _device_maps(db, cfg.TEST.SCALES[scale_id], rng)
        a_dev = CI.add_chips(db, maps, scale_id, cfg)
        a_host = CI.add_chips(dbh, host, scale_id, cfg)
        assert type(a_dev[0]) is type(a_host[0]) and np.array([a_dev]).tobytes() == np.array([a_host]).tobytes()
        for r, rh in zip(db, dbh):
            c, ch = r['inference_crops'], rh['inference_crops']
            assert c.dtype == ch.dtype and c.shape == ch.shape and c.tobytes() == ch.tobytes()
        if scale_id == 0:
            assert sum(len(r['inference_crops']) for r in db) >= len(db)
            db[3]['inference_crops'] = np.array([])                    # an image without chips at the next scale
            dbh[3]['inference_crops'] = np.array([])


def test_pyramid_device_chips_equal_host_chips_on_the_same_maps():
    """The fixture of test_pyramid_with_device_detections_equals_host_detections.  The device backend's pyramid is run
    scale by scale: at every scale that feeds a pruned scale, add_chips on the device maps object and on its host copies
    give the same chips and areas, and the host chips feed the next scale.  The final detections equal, byte for byte,
    those of imdb_detection_wrapper(detect_backend="device"), whose chips come from the device."""
    import torch
    from sniper_b200 import iterator as IT
    from sniper_b200 import model, synth_batch
    from sniper_b200 import tester as TS
    cfg = IT.default_config()
    cfg.TEST.SCALES = [(96, 160), (192, 320), (288, 480)]
    cfg.TEST.BATCH_IMAGES = [2, 2, 1]
    cfg.TEST.VALID_RANGES = [(40, -1), (16, 90), (-1, 40)]
    cfg.TEST.CHIP_HYPERPARAMS = [(3, 0.3, 4), (3, 0.4, 5)]
    rng = np.random.RandomState(2)
    db = [dict(width=W, height=H, image_data=rng.randint(0, 256, (H, W, 3)).astype(np.uint8))
          for (W, H) in ((320, 240), (240, 320), (300, 200))]
    mc = model.Cfg()
    mc.batch_images = 2
    net = model.SniperResNet101(mc, deform_offset_std=0.01)
    net.train_step(synth_batch.make_batch(2, seed=7, device="cuda"), lr=0.001)
    net.enable_autofocus(seed=3)
    boxes_d, stats_d = TS.imdb_detection_wrapper(net, cfg, db, detect_backend="device")
    chips_d = [np.array(r['inference_crops'], copy=True) for r in db]
    for r in db:
        r['inference_crops'] = np.array([[0, 0, r['width'], r['height']]])
    T, detections, compared = cfg.TEST, [], 0
    for scale_i, (nbatch, scale) in enumerate(zip(T.BATCH_IMAGES, T.SCALES)):
        it = TS.MNIteratorTestAutoFocus(db, cfg, scale, batch_size=nbatch)
        tester = TS.Tester(net, None, db, it, cfg, batch_size=nbatch)
        dets, maps = tester.get_detections(do_pruning=bool(T.DO_PRUNING[scale_i]), autofocus=bool(T.AUTO_FOCUS),
                                           backend="device", scale_index=scale_i)
        detections.append(dets)
        assert isinstance(maps, CI.DeviceFocusMaps)
        if scale_i + 1 < len(T.SCALES) and T.DO_PRUNING[scale_i + 1]:
            host = [[maps[i][j] for j in range(len(maps[i]))] for i in range(len(maps))]
            assert all(m[1].dtype == np.float32 and m[1].flags.c_contiguous for h in host for m in h)
            dbd = [dict(r) for r in db]
            a_dev = CI.add_chips(dbd, maps, scale_i, cfg)
            a_host = CI.add_chips(db, host, scale_i, cfg)
            assert np.array([a_dev]).tobytes() == np.array([a_host]).tobytes()
            for r, rd in zip(db, dbd):
                c, cd = r['inference_crops'], rd['inference_crops']
                assert c.dtype == cd.dtype and c.shape == cd.shape and c.tobytes() == cd.tobytes()
            compared += 1
    assert compared == 2
    for r, c in zip(db, chips_d):
        assert r['inference_crops'].tobytes() == c.tobytes()
    boxes = TS.Tester(net, None, db, None, cfg).aggregate(detections, backend="device")
    for j in range(1, 81):
        for i in range(3):
            assert boxes[j][i].dtype == boxes_d[j][i].dtype and boxes[j][i].tobytes() == boxes_d[j][i].tobytes()
    assert sum(len(boxes[j][i]) for j in range(1, 81) for i in range(3)) > 0
    torch.cuda.synchronize()
