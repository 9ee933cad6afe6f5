"""Proposal recall without a device: the numpy restatement (oracle/recall_np.py) against the reference's own
IMDB.evaluate_recall (tests/golden/recall_ref.npz, oracle/run_ref_recall.py), the host side of evaluate_recall, and the
argument checks of csrc/proposal_recall.cu.

The argument tests pass fabricated, never dereferenced device addresses (as test_voc_eval_cpu.py does): every call
violates one rule and must return from the check before any CUDA call."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", "oracle"))

import recall_fixture as F  # noqa: E402
import recall_np  # noqa: E402
from sniper_b200 import _lib, ops, recall  # noqa: E402

FAKE = 0x10000


@pytest.fixture(scope="module")
def fx():
    return F.load()


@pytest.mark.parametrize("name", F.CASES)
def test_restatement_equals_reference(fx, name):
    roidb, cand, thr, n_img = F.case(fx, name)
    text, rec, ov = F.expected(fx, name)
    got_text, got = recall_np.evaluate(roidb, cand, thr, n_img)
    assert got_text == text
    assert got['recalls'].tobytes() == rec.tobytes()
    for r in range(7):
        assert got['gt_overlaps'][r].tobytes() == ov[r].tobytes(), r


def test_reference_prints_what_it_returns(fx):
    for name in F.CASES:
        assert str(fx[name + '_stdout']).replace('\n', '') == str(fx[name + '_text'])


def test_golden_covers_the_rules(fx):
    roidb, cand, thr, n_img = F.case(fx, "hand")
    text, rec, ov = F.expected(fx, "hand")
    assert 'average recall for 300-inf: nan' in text          # num_pos == 0 (uint16 areas never reach 90000)
    assert 0.5 in ov[0] and 0.6 in ov[0]                       # IoUs equal to a default threshold
    assert 0.0 in ov[0]                                        # a round whose best overlap is 0
    assert np.dtype(roidb[0]['boxes'].dtype) == np.uint16 and cand[2].shape[0] == 0
    for name, T in (("thr1", 1), ("thr8", 8), ("thr9", 9), ("thr130", 130)):
        assert F.case(fx, name)[2].size == T
    merged = F.case(fx, "merged")
    assert merged[1] is None and merged[3] < len(merged[0]) and merged[0][0]['boxes'].dtype == np.float32


def test_host_masks_wrap_uint16_areas():
    g = np.array([[0, 0, 299, 299], [0, 0, 255, 255], [0, 0, 24, 24], [0, 0, 23, 24]], np.uint16)
    ov = np.zeros((4, 3), np.float32)
    ov[:, 1] = 1
    roidb = [{'boxes': g, 'gt_classes': np.ones(4, np.int32), 'gt_overlaps': ov}]
    prop_box, prop_off, gt_box, gt_off, gt_range = recall.recall_inputs(roidb, [np.zeros((0, 4), np.float32)])
    # 300 x 300 wraps to 24464 (100-200), 256 x 256 to 0 (0-25), 625 is in 25-50, 600 in 0-25
    assert list(gt_range) == [1 | 1 << 4, 1 | 1 << 1, 1 | 1 << 2, 1 | 1 << 1]
    assert gt_box.dtype == np.float64 and list(gt_off) == [0, 4] and list(prop_off) == [0, 0]


def test_host_refusals():
    ov = np.ones((1, 2), np.float32)
    e = {'boxes': np.array([[0, 0, 9, 9]], np.uint16), 'gt_classes': np.ones(1, np.int32), 'gt_overlaps': ov}
    with pytest.raises(ValueError, match="roidb has 1"):
        recall.recall_inputs([e], None, num_images=2)
    with pytest.raises(ValueError, match="candidate_boxes has 1"):
        recall.recall_inputs([e, e], [np.zeros((1, 4), np.float32)])
    with pytest.raises(ValueError, match="mix dtypes"):
        recall.recall_inputs([e, e], [np.ones((1, 4), np.float32), np.ones((1, 4), np.float64)])
    with pytest.raises(ValueError, match="thresholds"):
        recall.evaluate_recall([e], [np.ones((1, 4), np.float32)], thresholds=[1, 2])
    args = (np.zeros((1, 4), np.float32), [0, 1], np.zeros((1, 4)), [0, 1], [1], np.array([0.5]))
    with pytest.raises(ValueError, match="uint16, float32 or float64"):
        ops.proposal_recall(np.zeros((1, 4), np.int32), *args[1:])
    with pytest.raises(ValueError, match="finite"):
        ops.proposal_recall(np.full((1, 4), np.inf, np.float32), *args[1:])
    with pytest.raises(ValueError, match=r"\[N, 4\]"):
        ops.proposal_recall(np.zeros((2, 4), np.float32), *args[1:])
    with pytest.raises(ValueError, match="one mask per GT"):
        ops.proposal_recall(*args[:4], [1, 1], args[5])
    with pytest.raises(ValueError, match="1-D float64"):
        ops.proposal_recall(*args[:5], np.array([[0.5]]))


def test_restatement_refusals():
    # no proposal in any area range: the reference divides by zero
    g = {'boxes': np.array([[0, 0, 9, 9]]), 'gt_classes': np.ones(1, np.int32), 'gt_overlaps': np.ones((1, 2))}
    with pytest.raises(ValueError, match="no proposal"):
        recall_np.evaluate([g], [np.zeros((0, 4))])
    with pytest.raises(ValueError, match="index past"):
        recall_np.evaluate([g], [np.zeros((0, 4))], num_images=2)


def _c(v):
    return ctypes.c_void_p(v)


def test_workspace_bytes_checks():
    L = _lib.lib()
    off = np.array([0, 2], np.int32)
    bad = np.array([1, 2], np.int32)
    rng_ok = np.array([1, 1], np.uint8)
    ws = np.zeros(8, np.int64)
    assert L.sniper_proposal_recall_workspace_bytes(off.ctypes.data, off.ctypes.data, rng_ok.ctypes.data, 1,
                                                    ws.ctypes.data) == 0
    assert list(ws) == [0] * 8                                  # two proposals x one GT fit in shared memory
    assert L.sniper_proposal_recall_workspace_bytes(bad.ctypes.data, off.ctypes.data, rng_ok.ctypes.data, 1,
                                                    ws.ctypes.data) == -1
    assert b"prop_off" in L.sniper_last_error()
    assert L.sniper_proposal_recall_workspace_bytes(off.ctypes.data, off.ctypes.data,
                                                    np.array([1, 128], np.uint8).ctypes.data, 1, ws.ctypes.data) == -1
    assert b"bits above" in L.sniper_last_error()
    # 6000 proposals x 100 GTs: the worst case goes to the workspace
    big_p, big_g = np.array([0, 6000], np.int32), np.array([0, 100], np.int32)
    assert L.sniper_proposal_recall_workspace_bytes(big_p.ctypes.data, big_g.ctypes.data,
                                                    np.ones(100, np.uint8).ctypes.data, 1, ws.ctypes.data) == 0
    assert ws[1] == 6000 * 100 * 8 and ws[-1] == ws[1]


def test_match_and_accumulate_checks():
    L = _lib.lib()
    off = np.array([0, 2], np.int32)
    rng_ok = np.array([1, 1], np.uint8)
    ws = np.zeros(8, np.int64)
    args = [_c(FAKE), 1, _c(FAKE), _c(FAKE), _c(FAKE), _c(FAKE), _c(FAKE), _c(FAKE), off.ctypes.data, off.ctypes.data,
            rng_ok.ctypes.data, ws.ctypes.data, 1, 0, 7, None, _c(FAKE), _c(FAKE), None]
    a = list(args)
    a[1] = 3
    assert L.sniper_proposal_recall_match(*a) == -1 and b"prop_dtype" in L.sniper_last_error()
    a = list(args)
    a[14] = 8
    assert L.sniper_proposal_recall_match(*a) == -1 and b"must lie in" in L.sniper_last_error()
    a = list(args)
    a[13], a[14] = 3, 3
    assert L.sniper_proposal_recall_match(*a) == 0               # no pairs: no launch
    a = list(args)
    a[6] = None
    assert L.sniper_proposal_recall_match(*a) == -1 and b"must not be null" in L.sniper_last_error()
    ro = np.zeros(8, np.int64)
    npos = np.zeros(7, np.int64)
    acc = [_c(FAKE), ro.ctypes.data, npos.ctypes.data, _c(FAKE), 10, _c(FAKE), 1, 5, 1, _c(FAKE), _c(FAKE), _c(FAKE),
           _c(FAKE), _c(FAKE), None]
    a = list(acc)
    a[4] = -1
    assert L.sniper_proposal_recall_accumulate(*a) == -1 and b"thresholds" in L.sniper_last_error()
    a = list(acc)
    a[2] = np.array([0, 0, -1, 0, 0, 0, 0], np.int64).ctypes.data
    assert L.sniper_proposal_recall_accumulate(*a) == -1 and b"num_pos" in L.sniper_last_error()
    a = list(acc)
    a[1] = np.array([0, 5, 3, 3, 3, 3, 3, 3], np.int64).ctypes.data
    assert L.sniper_proposal_recall_accumulate(*a) == -1 and b"decrease" in L.sniper_last_error()


def test_header_and_bindings_carry_the_entry_points():
    hdr = open(os.path.join(HERE, "..", "include", "sniper_b200.h")).read()
    for name in ("sniper_proposal_recall_workspace_bytes", "sniper_proposal_recall_match",
                 "sniper_proposal_recall_accumulate"):
        assert re.search(r"\nint %s\(" % name, hdr), name
        assert name in _lib.SIGNATURES
    assert "proposal_recall.cu" in __import__("sniper_b200.build", fromlist=["NO_FMAD"]).NO_FMAD


def test_default_thresholds_are_numpys():
    t = recall.default_thresholds()
    assert t.size == 10 and t[2] == 0.6000000000000001 and t[2] != 0.6
