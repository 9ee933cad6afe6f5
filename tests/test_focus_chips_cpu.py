"""FocusChips on the device, the parts that need no device: the C-ABI declaration, the argument checks of
csrc/focus_chips.cu and `ops.focus_chips` (fabricated, never dereferenced addresses: every call breaks one rule and
must return before any CUDA call), and the table `DeviceFocusMaps` builds for the kernel against the values
`add_chips` / `gmask` / `Tester._chip_maps` compute, on batches of a host-only iterator."""
import math
import os

import numpy as np
import pytest
import torch

from sniper_b200 import _lib, ops
from sniper_b200 import chips_inference as CI
from sniper_b200 import iterator as IT
from sniper_b200 import tester as TS

HERE = os.path.dirname(os.path.abspath(__file__))
FAKE = 0x10000


def test_header_and_binding_declare_the_entry_points():
    h = open(os.path.join(HERE, "..", "include", "sniper_b200.h")).read()
    assert "int sniper_focus_chips_workspace_bytes(const long long* table_host, int n_maps, long long* ws_off_host);" in h
    assert ("int sniper_focus_chips(const long long* table, const long long* ws_off, const long long* table_host, "
            "const long long* ws_off_host, int n_maps, int d, float thresh, int ms, void* workspace, int cap, "
            "double* chips, int* counts, void* stream);") in h
    assert "lib/chips/chips_inference.py:12-89" in h
    assert _lib.SIGNATURES["sniper_focus_chips"] == ("i", "ppppiifipippp")
    assert _lib.SIGNATURES["sniper_focus_chips_workspace_bytes"] == ("i", "pip")
    assert _lib.KERNELS_PER_CALL["sniper_focus_chips_workspace_bytes"] == 0


def _table(H, W, n=1):
    t = np.zeros((n, ops.FOCUS_TABLE_COLS), np.int64)
    t[:, 0] = FAKE
    t[:, 1], t[:, 2] = 2 * W, 2
    t[:, 3], t[:, 4], t[:, 5], t[:, 6] = H, W, W, H
    t[:, 7:12] = np.array([W * 16.0, H * 16.0, 1.0, 0.0, 0.0]).view(np.int64)
    return t


def _call(t, ws_off=None, d=3, ms=4, cap=8, table=FAKE, workspace=None, chips=FAKE, counts=FAKE):
    L = _lib.lib()
    if ws_off is None:
        ws_off = np.zeros(len(t) + 1, np.int64)
        assert L.sniper_focus_chips_workspace_bytes(t.ctypes.data, len(t), ws_off.ctypes.data) == 0
    rc = L.sniper_focus_chips(table, FAKE, t.ctypes.data, ws_off.ctypes.data, len(t), d, 0.5, ms, workspace, cap, chips,
                              counts, None)
    return rc, L.sniper_last_error().decode()


def test_c_abi_refusals():
    L = _lib.lib()
    t = _table(20, 30)
    assert _call(t, d=0) == (-1, "focus_chips: the dilation size d (0) must be at least 1")
    assert "minimum chip size" in _call(t, ms=-1)[1]
    assert "cap" in _call(t, cap=-1)[1]
    assert "must not be null" in _call(t, table=None)[1]
    assert "must not be null" in _call(t, counts=None)[1]
    assert "chips must not be null" in _call(t, chips=None)[1]
    null = t.copy()
    null[0, 0] = 0
    assert "null address" in _call(null, np.zeros(2, np.int64))[1]
    neg = t.copy()
    neg[0, 3] = -1
    assert "cells" in _call(neg, np.zeros(2, np.int64))[1]
    big = _table(200, 200, 2)
    off = np.zeros(3, np.int64)
    assert L.sniper_focus_chips_workspace_bytes(big.ctypes.data, 2, off.ctypes.data) == 0
    assert off[1] == off[2] // 2 > 100 * 1024                           # too large for shared memory: one slice each
    assert "need a workspace" in _call(big, off)[1]
    assert "does not match" in _call(big, np.zeros(3, np.int64), workspace=FAKE)[1]
    assert L.sniper_focus_chips_workspace_bytes(t.ctypes.data, 1, None) == -1
    assert L.sniper_focus_chips_workspace_bytes(None, 1, off.ctypes.data) == -1


def test_ops_refusals():
    idx = np.array([[0, 0, 4, 5, 5, 4]], np.int64)
    geo = np.array([[80.0, 64.0, 1.0, 0.0, 0.0]])
    kw = dict(d=3, thresh=0.5, ms=4)
    cpu = torch.zeros(1, 4, 5)
    with pytest.raises(ValueError, match="float32"):
        ops.focus_chips([cpu], idx, geo, **kw)                            # not on a CUDA device
    with pytest.raises(ValueError, match="float32"):
        ops.focus_chips([cpu.double()], idx, geo, **kw)
    with pytest.raises(ValueError, match=r"\[n, 6\]"):
        ops.focus_chips([cpu], idx[:, :5], geo, **kw)
    with pytest.raises(ValueError, match="float64"):
        ops.focus_chips([cpu], idx, geo.astype(np.float32), **kw)
    with pytest.raises(ValueError, match="cscale"):
        ops.focus_chips([cpu], idx, geo * np.array([1, 1, 0, 1, 1]), **kw)
    with pytest.raises(ValueError, match="d"):
        ops.focus_chips([cpu], idx, geo, d=0, thresh=0.5, ms=4)
    with pytest.raises(ValueError, match="no tensor"):
        ops.focus_chips([], idx, geo, **kw)


def test_threshold_follows_numpy_promotion():
    v = np.float32(0.02)
    assert ops.focus_threshold(0.02) == v and (v >= 0.02)
    t = ops.focus_threshold(np.float64(0.02))                            # numpy compares this one in double
    assert not (v >= np.float64(0.02)) and not (v >= t) and np.nextafter(v, np.float32(1)) >= t
    assert ops.focus_threshold(1) == np.float32(1)


def test_table_of_a_host_only_iterator():
    cfg = IT.default_config()
    rng = np.random.RandomState(4)
    db = []
    for w, h in ((640, 480), (480, 640), (500, 333)):
        db.append(dict(width=w, height=h, image_data=rng.randint(0, 256, (h, w, 3)).astype(np.uint8),
                       inference_crops=np.array([[0.0, 0.0, w, h], [31.5, 12.25, w * 0.6, h * 0.7],
                                                 [w * 0.25, 40.0, w - 0.5, h - 3.0]])))
    db.append(dict(width=300, height=200, image_data=np.zeros((200, 300, 3), np.uint8),
                   inference_crops=np.array([[0, 0, 300, 200]])))          # an integer crop, as the first scale has
    scale = cfg.TEST.SCALES[1]
    it = TS.MNIteratorTestAutoFocus(db, cfg, scale, batch_size=4, device="cpu")
    maps = CI.DeviceFocusMaps([len(r['inference_crops']) for r in db], 16)
    last, batches = {}, []
    for k, b in enumerate(it):
        info = b['im_info'].numpy()
        Hc = int(math.ceil(info[:, 0].max() / 16))
        Wc = int(math.ceil(info[:, 1].max() / 16))
        fm = torch.from_numpy(rng.rand(len(info), Hc, Wc, 2).astype(np.float32))[..., 1]
        maps.add(fm, info, b['im_ids'], b['chip_ids'])
        batches.append((fm, info))
        for row, (i, j) in enumerate(zip(b['im_ids'], b['chip_ids'])):
            last[(int(i), int(j))] = (k, row)
    assert len(last) == sum(len(r['inference_crops']) for r in db) < it.size     # the iterator repeats crops
    index, geometry = maps.focus_table(db, scale)
    assert index.dtype == np.int64 and geometry.dtype == np.float64 and len(index) == len(last)
    m = 0
    tester = TS.Tester(None, None, db, None, cfg, num_classes=81)
    tester.net = type("N", (), {"feat_stride": 16})()
    for i, r in enumerate(db):
        cscale = CI.image_scale(r['width'], r['height'], scale)
        for j, crop in enumerate(r['inference_crops']):
            k, row = last[(i, j)]
            fm, info = batches[k]
            want = tester._chip_maps(fm.numpy(), info)[row]                # the map the host backend would hand gmask
            got = maps[i][j]
            assert got[0] is None and got[1].dtype == np.float32 and got[1].tobytes() == want.tobytes()
            assert got[1].shape == want.shape
            im_width, im_height = (crop[2] - crop[0]) * cscale, (crop[3] - crop[1]) * cscale
            assert list(index[m]) == [k, row, want.shape[0], want.shape[1], int(math.ceil(float(im_width) / 16)),
                                      int(math.ceil(float(im_height) / 16))]
            assert geometry[m].tobytes() == np.array([im_width, im_height, cscale, crop[0], crop[1]], np.float64).tobytes()
            m += 1
    assert len(maps) == len(db) and [len(maps[i]) for i in range(len(db))] == [3, 3, 3, 1]
    with pytest.raises(ValueError, match="crops"):
        maps.focus_table(db[:3] + [dict(db[3], inference_crops=np.zeros((2, 4)))], scale)
    empty = CI.DeviceFocusMaps([2], 16)
    assert empty[0][1] == [] and len(empty[0]) == 2
