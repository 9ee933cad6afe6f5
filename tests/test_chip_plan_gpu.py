"""The device epoch plan (chip_plan.DevicePlan, MNIteratorE2E(plan_backend="device")) is byte-equal to the host
chip_worker: positive chips as float64 bytes and tags, box-id arrays, negative chips and ids, and the C rand() position
after the plan; against tests/golden/chip_worker_ref.npz; and a whole iterator yields the same plans and raw batches."""
import copy
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from sniper_b200 import chip_plan, host
from sniper_b200 import chip_worker as CW
from sniper_b200 import iterator as IT

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
_libc = ctypes.CDLL(None)
DEV = "cuda:0"


def _host(cfg, roidb, stride, seed):
    cw = CW.chip_worker(cfg, 512)
    cw.chip_stride = cw.chip_generator.chip_stride = stride
    host.srand(seed)
    for r in roidb:
        r['crops'] = cw.chip_extractor(r)
    for r in roidb:
        ps = cw.box_assigner(r)
        r['props_in_chips'] = ps[0]
    return roidb, _libc.rand()


def _device(cfg, roidb, stride, seed, **kw):
    cw = CW.chip_worker(cfg, 512)
    cw.chip_stride = cw.chip_generator.chip_stride = stride
    plan = chip_plan.DevicePlan(roidb, cw, DEV, **kw)
    host.srand(seed)
    plan.plan(roidb)
    return roidb, _libc.rand()


def _same_chips(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.asarray(x[0], np.float64).tobytes() == np.asarray(y[0], np.float64).tobytes()
        assert x[1:] == y[1:] and [type(v) for v in x[1:]] == [type(v) for v in y[1:]]


def _same_lists(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()


def _compare(cfg, roidb, stride=58, seed=5, **kw):
    ref, r_after = _host(cfg, copy.deepcopy(roidb), stride, seed)
    got, g_after = _device(cfg, copy.deepcopy(roidb), stride, seed, **kw)
    assert g_after == r_after
    neg = cfg.TRAIN.USE_NEG_CHIPS
    for a, b in zip(ref, got):
        _same_chips(a['crops'], b['crops'])
        _same_lists(a['props_in_chips'], b['props_in_chips'])
        assert ('neg_chips' in b) == neg
        if neg:
            _same_chips(a['neg_chips'], b['neg_chips'])
            _same_lists(a['neg_props_in_chips'], b['neg_props_in_chips'])
    return ref


def _roidb(n, seed, **kw):
    return [{k: v for k, v in r.items() if k != 'image_data'} for r in IT.synthetic_roidb(n, seed=seed, **kw)]


@pytest.mark.parametrize("neg", [False, True])
@pytest.mark.parametrize("scales", ["coco", "paper", "voc"])
def test_device_plan_equals_chip_worker(neg, scales):
    cfg = IT.default_config(neg=neg, dataset="pascal_voc" if scales == "voc" else "coco")
    if scales == "paper":
        cfg.TRAIN.SCALES = (3.0, 1.667, 512.0)
    roidb = _roidb(6, 1, n_prop=300 if neg else 0)
    roidb += _roidb(3, 2, width=400, height=300, n_prop=500 if neg else 0)       # smaller than a chip at some scales
    ref = _compare(cfg, roidb, stride=56 + len(scales))
    assert sum(len(r['crops']) for r in ref) > 0
    if neg:
        assert sum(len(r['neg_chips']) for r in ref) > 0


def test_flipped_entries_empty_entries_and_uint16_boxes():
    cfg = IT.default_config(neg=True)
    roidb = _roidb(4, 3, n_prop=400)
    for r in list(roidb):                                       # load_data.append_flipped_images
        b = r['boxes'].copy()
        b[:, 0], b[:, 2] = r['width'] - r['boxes'][:, 2] - 1, r['width'] - r['boxes'][:, 0] - 1
        roidb.append(dict(r, boxes=b, flipped=True))
    no_gt = dict(roidb[0], max_overlaps=np.minimum(roidb[0]['max_overlaps'], 0.5))
    empty = dict(roidb[1], boxes=roidb[1]['boxes'][:0], max_overlaps=roidb[1]['max_overlaps'][:0])
    u16 = dict(roidb[2], boxes=np.round(roidb[2]['boxes']).astype(np.uint16))
    u16['boxes'][0] = [50, 40, 30, 60]                          # x2 < x1: the uint16 width wraps, as on the host
    _compare(cfg, roidb + [no_gt, empty, u16])


def test_duplicate_boxes_and_tied_counts():
    cfg = IT.default_config(neg=True)
    rng = np.random.RandomState(4)
    roidb = []
    for k in range(4):
        base = np.array([[100, 100, 160, 150], [700, 300, 790, 380], [10, 600, 40, 640]], np.float32)
        props = np.repeat(base, 20, axis=0) + rng.randint(0, 3, (60, 4)).astype(np.float32)
        boxes = np.concatenate([base, base, props])
        mo = np.concatenate([np.ones(6), np.full(60, 0.3)]).astype(np.float32)
        roidb.append(dict(width=1333, height=800, boxes=boxes, max_overlaps=mo, flipped=False))
    _compare(cfg, roidb)


def test_workspace_path_chunks_and_uploads():
    cfg = IT.default_config(neg=True)
    roidb = _roidb(3, 6, width=2000, height=1500, n_prop=3000)
    roidb += _roidb(4, 7, n_prop=200)
    _compare(cfg, roidb, chunk_images=2, resident_bytes=0)
    cw = CW.chip_worker(cfg, 512)
    plan = chip_plan.DevicePlan(roidb, cw, DEV, chunk_images=2)
    nb = np.diff(plan.box_off)
    n_cand = chip_plan.n_candidates(plan.W, plan.H, 512, cw.chip_stride)
    words = (nb[:, None] + 63) // 64
    assert (8 * n_cand * words > 64 * 1024).any()              # some cover's scratch exceeds shared memory


def test_committed_golden():
    import run_ref_chip_worker as RR
    from test_chip_worker_cpu import CASES, _flatten
    gold = np.load(os.path.join(ROOT, "tests", "golden", "chip_worker_ref.npz"))
    for ci, case in enumerate(CASES):
        cfg = RR.make_cfg(**case["cfg"])
        r = dict(RR.synth_roidb(case["seed"], **case["roidb"]))
        (r,), _ = _device(cfg, [r], 58, 1 + case["seed"])
        out = (r['props_in_chips'], r['neg_chips'], r['neg_props_in_chips']) if cfg.TRAIN.USE_NEG_CHIPS else \
            (r['props_in_chips'],)
        for k, v in _flatten(r['crops'], out).items():
            g = gold["c%d_%s" % (ci, k)]
            assert g.shape == v.shape and g.tobytes() == v.tobytes(), (ci, k)


def _raw_bytes(raw):
    keys = ("table", "valid_ranges", "im_info", "gt_valid", "ngt", "gt_invalid", "ninv", "gt_boxes", "anchor_im_info")
    return b"".join(getattr(raw, k).numpy().tobytes() for k in keys) + raw.pixels[:raw.used_pixels].numpy().tobytes()


def _epochs(backend, seed, rank, nGPUs):
    cfg = IT.default_config(neg=True)
    roidb = IT.synthetic_roidb(5, seed=11, width=600, height=450, n_prop=300)
    np.random.seed(3)
    host.srand(17)
    it = IT.MNIteratorE2E(roidb, cfg, batch_size=4, nGPUs=nGPUs, rank=rank, seed=seed, plan_backend=backend,
                          device=DEV if backend == "device" else None)
    out = []
    for ep in range(2):
        if ep:
            it.reset()
        out.append((it.plan_digest, len(it), [_raw_bytes(raw) for raw in it]))
    return out, _libc.rand(), np.random.randint(1 << 30)


@pytest.mark.parametrize("seed", [None, 5])
def test_iterator_device_backend_equals_host(seed):
    for rank, nGPUs in [(None, 1)] + ([(0, 2), (1, 2)] if seed is not None else []):
        h = _epochs("host", seed, rank, nGPUs)
        d = _epochs("device", seed, rank, nGPUs)
        assert d[1:] == h[1:]
        for (hd, hl, hb), (dd, dl, db) in zip(h[0], d[0]):
            assert dd == hd and dl == hl and db == hb
