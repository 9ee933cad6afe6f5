"""The inference proposal operator (ops.multi_proposal -> sniper_multi_proposal_fwd) byte-equal to oracle/mp_cpuop.c at
the geometry the Tester runs: rectangular canvases of both graphs (stride 16 / 21 anchors / 12000 pre-NMS rows and
stride 32 / 15 anchors / 6000), per-image im_info smaller than the canvas, NCHW, NHWC and the graph's own padded head,
score regimes with exact ties (quantised logits, a saturated softmax, a run across the pre-NMS rank K, a run longer than
a trip of the bit-mask NMS), filler rows, anchor-type suppression and FastNMS.  Every case runs on the bit-mask NMS and
on the sequential kernel (SNIPER_NMS_FAST=1 / 0).  Inputs: tests/multi_proposal_cases.py."""
import functools

import numpy as np
import pytest

import multi_proposal_cases as C
import oracle_lib as O

pytestmark = pytest.mark.gpu


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@functools.lru_cache(maxsize=None)
def _oracle(name):
    c = C.build(name)
    return O.multi_proposal(c["cls_prob"], c["bbox_pred"], c["im_info"], pre=c["pre"], flags=c["flags"],
                            roi_iou_thresh=0.3, libm_exp=False, **c["kw"])


def _device(monkeypatch, fast, cls_prob, bbox_pred, im_info, layout="nchw", flags=0, **kw):
    import torch
    from sniper_b200 import ops
    monkeypatch.setenv("SNIPER_NMS_FAST", fast)
    out = ops.multi_proposal(_t(cls_prob), _t(bbox_pred), _t(im_info), suppress_anchor_types=bool(flags & 1),
                             fast_nms=bool(flags & 2), roi_iou_thresh=0.3,
                             layout=ops.NCHW if layout == "nchw" else ops.NHWC, return_keep=True, return_fallback=True,
                             **kw)
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in out]


def _assert_equal(got, ref):
    rois, scores, keep, nk = got[:4]
    np.testing.assert_array_equal(nk, ref["num_kept"])
    np.testing.assert_array_equal(keep, ref["keep_idx"])
    assert rois.tobytes() == ref["rois"].tobytes()          # filler rows included
    assert scores.tobytes() == ref["scores"].tobytes()


@pytest.mark.parametrize("fast", ["1", "0"])
@pytest.mark.parametrize("name", C.CASE_NAMES)
def test_multi_proposal_byte_equal_to_oracle_at_tester_canvases(name, fast, monkeypatch):
    c = C.build(name)
    ref = _oracle(name)
    prob, bbox = C.device_inputs(c["cls_prob"], c["bbox_pred"], c["layout"], c["head_c"])
    got = _device(monkeypatch, fast, prob, bbox, c["im_info"], c["layout"], c["flags"], rpn_pre_nms_top_n=c["pre"],
                  **c["kw"])
    _assert_equal(got, ref)
    if c["filler"]:
        assert ref["num_kept"][-1] < 300 and (ref["num_kept"][:-1] == 300).all()
    if fast == "1":
        fb = got[4]
        if c["regime"] in ("tie_free", "quantised", "strip_pairs"):
            assert (fb == 0).all(), "the bit-mask NMS fell back: %s" % fb      # its own tie handling is what ran
        elif c["regime"] in ("saturated", "long_run", "k_boundary"):
            assert (fb == 1).all(), "the bit-mask NMS did not fall back: %s" % fb


@pytest.mark.parametrize("fast", ["1", "0"])
def test_multi_proposal_tied_rows_are_kept_in_index_order(fast, monkeypatch):
    """Two equal top scores at rows 1 and 32 with disjoint boxes: both are kept, row 1 first (the scan order of the
    training operator's NMS would take row 32, lane 0 of warp 1, before row 1, lane 1 of warp 0)."""
    cls_prob, bbox_pred, im_info, (i, j) = C.tied_pair(overlap=False)
    ref = O.multi_proposal(cls_prob, bbox_pred, im_info, libm_exp=False)
    assert list(ref["keep_idx"][:2]) == [i, j]
    got = _device(monkeypatch, fast, cls_prob, bbox_pred, im_info)
    assert list(got[2][:2]) == [i, j]
    _assert_equal(got, ref)
    if fast == "1":
        assert (got[4] == 0).all()


@pytest.mark.parametrize("fast", ["1", "0"])
def test_multi_proposal_overlapping_tie_keeps_the_lower_index(fast, monkeypatch):
    """Rows 5 and 1026 share the top score and the same box: row 5 is kept, row 1026 suppressed."""
    cls_prob, bbox_pred, im_info, (i, j) = C.tied_pair(overlap=True)
    ref = O.multi_proposal(cls_prob, bbox_pred, im_info, libm_exp=False)
    assert ref["keep_idx"][0] == i and j not in ref["keep_idx"]
    got = _device(monkeypatch, fast, cls_prob, bbox_pred, im_info)
    assert got[2][0] == i and j not in got[2]
    _assert_equal(got, ref)
    if fast == "1":
        assert (got[4] == 0).all()
