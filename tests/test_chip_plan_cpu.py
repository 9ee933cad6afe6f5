"""The device epoch plan (csrc/chip_plan.cu, sniper_b200/chip_plan.py), the parts that need no device.

- `sniper_chips_shuffle` draws from rand() what a sequence of `host.chips_generate` calls draws: a numpy greedy cover over
  its permutation reproduces `host.chips_generate` chip for chip, rand() ends at the same position, and calls without
  boxes draw nothing.
- A numpy restatement of the device plan's phase split (positive counts -> draws -> covers -> assignment -> negative
  counts -> draws -> covers -> assignment) equals `chip_worker` on seeded roidbs, rand() position included.
- The C-ABI entry points refuse bad arguments before any CUDA call (fabricated, never dereferenced addresses)."""
import ctypes
import os

import numpy as np
import pytest

from sniper_b200 import _lib, build, chip_plan, host
from sniper_b200 import chip_worker as CW
from sniper_b200 import iterator as IT

HERE = os.path.dirname(os.path.abspath(__file__))
_libc = ctypes.CDLL(None)
FAKE = 0x7f0000100000


def _rand():
    return _libc.rand()


def _candidates(W, H, cs, s):
    """sniper_chips_generate's candidates in push order, float32 [n, 4]."""
    c = [(max(W - cs, 0), 0, W - 1, min(cs, H - 1)), (0, max(H - cs, 0), min(cs, W - 1), H - 1),
         (max(W - cs, 0), max(H - cs, 0), W - 1, H - 1)]
    c += [(i, j, i + cs - 1, j + cs - 1) for i in range(0, W - cs, s) for j in range(0, H - cs, s)]
    c += [(max(W - cs - 1, 0), i, W - 1, i + cs - 1) for i in range(0, H - cs, s)]
    c += [(i, max(H - cs - 1, 0), i + cs - 1, H - 1) for i in range(0, W - cs, s)]
    return np.array(c, np.float32)


def _greedy(boxes, W, H, cs, s, perm):
    """chips_generate's greedy cover over the candidate order `perm`, in numpy float32."""
    cand = _candidates(W, H, cs, s)[perm]
    b = np.asarray(boxes, np.float32).reshape(-1, 4)
    one = np.float32(1)
    area2 = (b[:, 2] - b[:, 0] + one) * (b[:, 3] - b[:, 1] + one)
    iw = np.minimum(cand[:, None, 2], b[None, :, 2]) - np.maximum(cand[:, None, 0], b[None, :, 0]) + one
    ih = np.minimum(cand[:, None, 3], b[None, :, 3]) - np.maximum(cand[:, None, 1], b[None, :, 1]) + one
    with np.errstate(divide="ignore", invalid="ignore"):
        match = (iw > 0) & (ih > 0) & (iw * ih / area2[None, :] == one)
    out = []
    while True:
        cnt = match.sum(1)
        if cnt.max(initial=0) == 0:
            break
        k = int(np.argmax(cnt))
        out.append(cand[k])
        match &= ~match[k][None, :]
    return np.array(out, np.float32).reshape(-1, 4)


def _scaled(boxes, f, W, H):
    b = np.array(boxes * f, dtype=np.float64).reshape(-1, 4)
    b[:, 0::2] = np.maximum(np.minimum(b[:, 0::2], W - 2), 0)
    b[:, 1::2] = np.maximum(np.minimum(b[:, 1::2], H - 2), 0)
    return b.astype(np.float32)


def test_n_candidates_matches_the_push_order():
    for W, H, cs, s in [(2333, 1400, 512, 56), (512, 512, 512, 59), (300, 900, 512, 57), (1, 1, 512, 58), (513, 600, 512, 3)]:
        assert chip_plan.n_candidates(W, H, cs, s) == len(_candidates(W, H, cs, s))


def test_shuffle_reproduces_chips_generate_and_the_rand_position():
    rng = np.random.RandomState(0)
    calls = []
    for k in range(12):
        W, H = int(rng.randint(200, 2500)), int(rng.randint(200, 2500))
        nb = 0 if k % 4 == 1 else int(rng.randint(1, 60))
        x1, y1 = rng.uniform(0, W, nb), rng.uniform(0, H, nb)
        b = np.stack([x1, y1, x1 + rng.uniform(4, 400, nb), y1 + rng.uniform(4, 400, nb)], 1)
        calls.append((_scaled(b, 1.0, W, H), W, H))
    stride = 57
    host.srand(123)
    ref = [host.chips_generate(b, W, H, 512, stride) for b, W, H in calls]
    after_host = _rand()
    host.srand(123)
    n_cand = [chip_plan.n_candidates(W, H, 512, stride) if len(b) else 0 for b, W, H in calls]
    perm = chip_plan.chips_shuffle(n_cand)
    after_shuffle = _rand()
    assert after_shuffle == after_host
    off = 0
    for (b, W, H), n, want in zip(calls, n_cand, ref):
        if n == 0:
            assert len(want) == 0
            continue
        got = _greedy(b, W, H, 512, stride, perm[off:off + n])
        off += n
        assert got.tobytes() == want.tobytes()


def test_calls_without_boxes_draw_nothing():
    host.srand(7)
    assert len(host.chips_generate(np.zeros((0, 4), np.float32), 900, 700, 512, 58)) == 0
    a = _rand()
    host.srand(7)
    chip_plan.chips_shuffle([0, 0, 0])
    assert _rand() == a
    host.srand(7)
    first = _rand()
    assert first == a


def _restated_plan(cw, roidb):
    """The device plan's phase split in numpy: which calls draw follows from the positive counts, then from the boxes
    no positive chip kept; every positive draw comes before every negative one."""
    S = len(cw.scales)
    cs, st = cw.chip_size, cw.chip_stride
    geo, pos_boxes = [], []
    for r in roidb:
        fs = CW.image_scales(cw.scales, r['width'], r['height'])
        gt = r['boxes'][np.where(r['max_overlaps'] == 1)[0], :]
        w, h, size, longest = cw._int_sizes(gt)
        for i, f in enumerate(fs):
            lo, hi = cw.valid_ranges[i]
            if i == S - 1:
                sel = size >= lo
            elif i == 0:
                sel = (size < hi) & cw._fits(longest, f) & (w >= 2) & (h >= 2)
            else:
                sel = (size >= lo) & (size < hi) & cw._fits(longest, f)
            W, H = int(r['width'] * f), int(r['height'] * f)
            geo.append((f, W, H))
            pos_boxes.append(_scaled(gt[np.where(sel)[0], :] * f, 1.0, W, H))
    n_cand = [chip_plan.n_candidates(W, H, cs, st) if len(b) else 0 for (f, W, H), b in zip(geo, pos_boxes)]
    perm = chip_plan.chips_shuffle(n_cand)
    offs = np.cumsum([0] + n_cand)
    chips = [_greedy(b, W, H, cs, st, perm[offs[c]:offs[c + 1]])[:chip_plan.HOST_CAP] if len(b) else np.zeros((0, 4))
             for c, (b, (f, W, H)) in enumerate(zip(pos_boxes, geo))]
    left_all, out = [], []
    for e, r in enumerate(roidb):
        crops = []
        for i in range(S):
            f = geo[e * S + i][0]
            crops += [cw._tag(c, f, i, r) for c in np.array(chips[e * S + i], np.float64) / f]
        w, h, size, longest = cw._int_sizes(r['boxes'])
        props = [None] * len(crops)
        base = 0
        for i in range(S):
            f = geo[e * S + i][0]
            if i == S - 1:
                ids = np.where(size >= cw.valid_ranges[i][0])[0]
            else:
                ids = np.where((size < cw.valid_ranges[i][1]) & cw._fits(longest, f) & (w >= 2) & (h >= 2))[0]
            ch = np.array(chips[e * S + i], np.float64) / f
            per_chip, kept = cw._assign(ch, r['boxes'][ids].astype(float), ids, i, strict_hi=False)
            for k, lst in enumerate(per_chip):
                props[base + k] = np.array(lst, np.int32)
            base += len(ch)
            left_all.append((r['boxes'][ids].astype(float)[~kept], ids[~kept]))
        out.append((crops, props))
    n_cand = [chip_plan.n_candidates(W, H, cs, st) if len(lb) else 0 for (f, W, H), (lb, _) in zip(geo, left_all)]
    perm = chip_plan.chips_shuffle(n_cand)
    offs = np.cumsum([0] + n_cand)
    res = []
    for e, r in enumerate(roidb):
        neg_c, neg_p = [], []
        for i in range(S):
            c = e * S + i
            f, W, H = geo[c]
            lb, lid = left_all[c]
            nc = (_greedy(_scaled(lb * f, 1.0, W, H), W, H, cs, st, perm[offs[c]:offs[c + 1]])[:chip_plan.HOST_CAP]
                  if len(lb) else np.zeros((0, 4)))
            ch = np.array(nc, np.float64) / f
            per_chip, _ = cw._assign(ch, lb, lid, i, strict_hi=True)
            for cc, lst in zip(ch, per_chip):
                if len(lst) > 25 or (len(lst) > 10 and i != 0):
                    neg_c.append(cw._tag(cc, f, i, r))
                    neg_p.append(np.array(lst, dtype=int))
        res.append(out[e] + (neg_c, neg_p))
    return res


def _same_chips(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.asarray(x[0], np.float64).tobytes() == np.asarray(y[0], np.float64).tobytes()
        assert x[1:] == y[1:]


def _same_lists(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and x.tobytes() == y.tobytes()


@pytest.mark.parametrize("scales", ["coco", "paper"])
def test_restated_phase_split_equals_chip_worker(scales):
    cfg = IT.default_config(neg=True)
    if scales == "paper":
        cfg.TRAIN.SCALES = (3.0, 1.667, 512.0)
    roidb = IT.synthetic_roidb(5, seed=3, width=700, height=500, n_prop=250)
    roidb.append(dict(roidb[0], boxes=roidb[0]['boxes'][:0], max_overlaps=roidb[0]['max_overlaps'][:0]))
    cw = CW.chip_worker(cfg, 512, rng=np.random.RandomState(1))
    host.srand(99)
    ref = []
    for r in roidb:
        r['crops'] = cw.chip_extractor(r)
    for r in roidb:
        ps = cw.box_assigner(r)
        ref.append((r['crops'], ps[0], ps[1], ps[2]))
    after = _rand()
    host.srand(99)
    got = _restated_plan(cw, roidb)
    assert _rand() == after
    assert sum(len(x[2]) for x in ref) > 0
    for (c, p, nc, npr), (c2, p2, nc2, np2) in zip(ref, got):
        _same_chips(c, c2)
        _same_lists(p, p2)
        _same_chips(nc, nc2)
        _same_lists(npr, np2)


def test_chip_plan_is_built_without_fma():
    assert "chip_plan.cu" in build.NO_FMAD


def test_header_and_binding_declare_the_entry_points():
    h = open(os.path.join(HERE, "..", "include", "sniper_b200.h")).read()
    assert "int sniper_chips_shuffle(const int* n_cand, int n_calls, int* perm_out);" in h
    for name in ("sniper_chip_plan_layout", "sniper_chip_plan_count", "sniper_chip_plan_cover",
                 "sniper_chip_plan_assign"):
        assert "int %s(" % name in h
    assert _lib.KERNELS_PER_CALL["sniper_chips_shuffle"] == 0 and _lib.KERNELS_PER_CALL["sniper_chip_plan_layout"] == 0


def _table(n=1, W=900, H=700, nbox=5, cs=512, stride=58):
    t = np.zeros((n, chip_plan.TABLE_COLS), np.int64)
    t[:, chip_plan.C_SCALE] = 0
    t[:, chip_plan.C_KIND] = 2
    t[:, chip_plan.C_W], t[:, chip_plan.C_H] = W, H
    t[:, chip_plan.C_NCAND] = chip_plan.n_candidates(W, H, cs, stride)
    t[:, chip_plan.C_NBOX] = nbox
    t[:, chip_plan.C_CAP] = min(int(t[0, chip_plan.C_NCAND]), nbox)
    t[:, chip_plan.C_F] = np.array([1.0]).view(np.int64)[0]
    ws = np.zeros(1, np.int64)
    assert _lib.lib().sniper_chip_plan_layout(t.ctypes.data, n, cs, stride, ws.ctypes.data) == 0
    return t


def _cover(t, **kw):
    a = dict(table=FAKE, n_calls=len(t), mode=0, S=1, cs=512, stride=58, box_off=FAKE, boxes=FAKE, wh=FAKE, gt=FAKE,
              pos_owner=None, perm=FAKE, ws=None, ws_bytes=0, chips32=FAKE, chips64=FAKE, nchips=FAKE)
    a.update(kw)
    L = _lib.lib()
    rc = L.sniper_chip_plan_cover(a["table"], t.ctypes.data, a["n_calls"], a["mode"], a["S"], a["cs"], a["stride"],
                                  a["box_off"], a["boxes"], a["wh"], a["gt"], a["pos_owner"], a["perm"], a["ws"],
                                  a["ws_bytes"], a["chips32"], a["chips64"], a["nchips"], None)
    return rc, L.sniper_last_error().decode()


@pytest.mark.parametrize("change, pattern", [
    (dict(mode=2), "mode"),
    (dict(mode=1), "pos_owner"),
    (dict(gt=None), "needs gt"),
    (dict(perm=None), "must not be null"),
    (dict(S=0), "scale count"),
    (dict(stride=0), "stride"),
    (dict(stride=60), "n_cand"),
    (dict(boxes=FAKE + 4), "aligned"),
    (dict(chips64=FAKE + 16), "aligned"),
])
def test_cover_refuses_bad_arguments(change, pattern):
    rc, msg = _cover(_table(W=2000), **change)
    assert rc == -1 and pattern in msg, msg


def test_cover_refuses_a_table_it_did_not_lay_out():
    t = _table(nbox=2000, W=3000, H=3000)
    assert t[0, chip_plan.C_WS] == 0                       # past the shared-memory cap: a workspace slice
    rc, msg = _cover(t)
    assert rc == -1 and "workspace" in msg, msg
    t2 = _table()
    t2[0, chip_plan.C_WS] = 0
    rc, msg = _cover(t2)
    assert rc == -1 and "sniper_chip_plan_layout" in msg, msg
    t3 = _table()
    t3[0, chip_plan.C_CAP] = 1
    rc, msg = _cover(t3)
    assert rc == -1 and "output slots" in msg, msg


def test_count_and_assign_refuse_bad_arguments():
    L = _lib.lib()
    t = _table()
    assert L.sniper_chip_plan_count(FAKE, t.ctypes.data, 1, 1, 512, 58, FAKE, FAKE, None, FAKE, None) == -1
    assert "must not be null" in L.sniper_last_error().decode()
    t[0, chip_plan.C_SCALE] = 3
    assert L.sniper_chip_plan_count(FAKE, t.ctypes.data, 1, 1, 512, 58, FAKE, FAKE, FAKE, FAKE, None) == -1
    assert "bad entry / scale / kind" in L.sniper_last_error().decode()
    t = _table()
    assert L.sniper_chip_plan_assign(FAKE, t.ctypes.data, 1, 1, 1, FAKE, FAKE, FAKE, None, FAKE, FAKE, FAKE, FAKE,
                                     None) == -1
    assert "pos_owner" in L.sniper_last_error().decode()
    assert L.sniper_chip_plan_assign(FAKE, t.ctypes.data, 1, 0, 1, FAKE, FAKE + 8, FAKE, None, FAKE, FAKE, FAKE, FAKE,
                                     None) == -1
    assert "aligned" in L.sniper_last_error().decode()


def test_shuffle_refuses_before_drawing():
    L = _lib.lib()
    n = np.array([5, -1], np.int32)
    out = np.zeros(8, np.int32)
    host.srand(5)
    assert L.sniper_chips_shuffle(n.ctypes.data, 2, out.ctypes.data) == -1
    assert "candidates" in L.sniper_last_error().decode()
    a = _rand()
    host.srand(5)
    assert _rand() == a
    n = np.array([4], np.int32)
    assert L.sniper_chips_shuffle(n.ctypes.data, 1, None) == -1


def test_iterator_refuses_an_unknown_backend():
    with pytest.raises(ValueError, match="plan_backend"):
        IT.MNIteratorE2E(IT.synthetic_roidb(1, n_prop=0), IT.default_config(neg=False), batch_size=1,
                         plan_backend="gpu")
