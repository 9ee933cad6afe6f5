"""The inputs of tests/test_multi_proposal_exact_gpu.py are what they claim (tests/multi_proposal_cases.py): Tester
geometry of both graphs, the tie regimes, the graph layout's NaN padding, filler rows and the hand-built tie cases --
checked here, on the oracle, without a GPU."""
import functools

import numpy as np
import pytest

import multi_proposal_cases as C
import oracle_lib as O


@functools.lru_cache(maxsize=None)
def _oracle(name):
    c = C.build(name)
    return O.multi_proposal(c["cls_prob"], c["bbox_pred"], c["im_info"], pre=c["pre"], flags=c["flags"],
                            roi_iou_thresh=0.3, libm_exp=False, **c["kw"])


def _fg(c):
    B, A = c["cls_prob"].shape[0], c["A"]
    return c["cls_prob"][:, A:].reshape(B, -1)


def test_graph_parameters_come_from_the_networks():
    r, m = C.graph("resnet101"), C.graph("mobilenetv2")
    assert (r["feat_stride"], r["A"], r["pre"], r["head_c"]) == (16, 21, 12000, 128)
    assert (m["feat_stride"], m["A"], m["pre"], m["head_c"]) == (32, 15, 6000, 96)


def test_geometry_covers_the_tester_canvases():
    cases = [C.build(n) for n in C.CASE_NAMES]
    for network in C.NETWORKS:
        mine = [c for c in cases if c["network"] == network]
        assert {c["scale_i"] for c in mine} == {0, 1, 2}
        assert {c["layout"] for c in mine} == {"nchw", "nhwc", "graph"}
        assert {c["regime"] for c in mine} >= {"tie_free", "quantised", "saturated", "k_boundary", "long_run"}
        assert {c["flags"] for c in mine} == {0, 1, 2, 3}
        assert any(c["A"] * c["H"] * c["W"] < c["pre"] for c in mine) or network == "resnet101"
    assert max(c["A"] * c["H"] * c["W"] for c in cases) > 200000                    # the largest ResNet-101 canvas
    assert any(c["A"] * c["H"] * c["W"] < c["pre"] for c in cases)                 # no pre-NMS selection
    for c in cases:
        stride = c["kw"]["feat_stride"]
        info = c["im_info"]
        assert c["H"] != c["W"] or c["scale_i"] == 2
        assert (info[:, 0] <= c["H"] * stride).all() and (info[:, 1] <= c["W"] * stride).all()
        assert (info[:, 0] != info[:, 1]).all()                                    # h != w in every image
        assert (info[:, 0] < c["H"] * stride).any() or (info[:, 1] < c["W"] * stride).any()
        assert len(np.unique(info[:, :2], axis=0)) > 1                             # per-image im_info differs
        assert c["cls_prob"].shape == (len(info), 2 * c["A"], c["H"], c["W"])
        assert c["bbox_pred"].shape == (len(info), 4 * c["A"], c["H"], c["W"])
    # the 1333 x 800 image at the largest test scale: a 1216 x 2048 canvas as in the Tester
    assert C.tester_batch("resnet101", 2, [(1333, 800)])[1:] == (76, 128)
    assert C.tester_batch("mobilenetv2", 0, [(1333, 800)])[1:] == (38, 64)


def test_graph_layout_pads_the_head_with_nan():
    c = C.build("resnet101-s0-landscape")
    prob, head = C.device_inputs(c["cls_prob"], c["bbox_pred"], "graph", c["head_c"])
    A = c["A"]
    assert prob.shape == c["cls_prob"].transpose(0, 2, 3, 1).shape and prob.flags.c_contiguous
    assert head.shape[3] == 128 and head.flags.c_contiguous
    assert np.array_equal(head[..., :4 * A], c["bbox_pred"].transpose(0, 2, 3, 1))
    assert np.isnan(head[..., 4 * A:]).all()
    nhwc = C.device_inputs(c["cls_prob"], c["bbox_pred"], "nhwc", c["head_c"])[1]
    assert nhwc.shape[3] == 4 * A


def _runs_at_top(fg_row, top):
    v = np.sort(fg_row)[::-1][:top]
    _, counts = np.unique(v, return_counts=True)
    return counts


def test_tie_regimes():
    c = C.build("resnet101-largest-saturated")
    fg = _fg(c)
    for b in range(len(fg)):
        assert (fg[b] == np.float32(1.0)).sum() >= 1000 and (fg[b] == C.ONE_BELOW_ONE).sum() >= 1000
    for name in ("resnet101-largest-quantised", "mobilenetv2-largest-quantised", "resnet101-s1-landscape"):
        c = C.build(name)
        for row in _fg(c):
            counts = _runs_at_top(row, 4096)            # the bit-mask NMS's candidates
            assert (counts > 1).sum() > 100 and counts.max() <= 64, (name, counts.max())
    for name in ("resnet101-largest-long_run", "mobilenetv2-largest-long_run", "mobilenetv2-small-long_run"):
        for row in _fg(C.build(name)):
            v = np.sort(row)[::-1]
            assert len(np.unique(v[:10])) == 10 and (v[10:110] == v[10]).all() and v[110] < v[10]
    c = C.build("mobilenetv2-small-long_run")
    assert c["A"] * c["H"] * c["W"] < c["pre"]


@pytest.mark.parametrize("name", ["resnet101-largest-k_boundary", "mobilenetv2-largest-k_boundary"])
def test_k_boundary_run_straddles_the_selection(name):
    c = C.build(name)
    K = c["pre"]
    ref = _oracle(name)
    A, H, W = c["A"], c["H"], c["W"]
    dw = c["bbox_pred"].reshape(-1, A, 4, H * W)[:, :, 2].reshape(len(c["im_info"]), -1)
    for b, row in enumerate(_fg(c)):
        v = np.sort(row)[::-1]
        assert v[K - 41] > v[K - 40] == v[K - 1] == v[K] == v[K + 59] > v[K + 60]
        run = np.flatnonzero(row == v[K])
        assert (dw[b][row > v[K]] == C.BIG_DELTA).all()
        kept = ref["keep_idx"][b * 300:b * 300 + ref["num_kept"][b]]
        # one whole-image box, then only rows of the run -- the 40 of lowest index that the selection admits
        assert (row[kept[0]] > v[K]) and (row[kept[1:]] == v[K]).all() and len(kept) > 10
        assert set(kept[1:]) <= set(run[:40]) and not set(kept[1:]) & set(run[40:])


@pytest.mark.parametrize("name", ["resnet101-mid-filler", "mobilenetv2-mid-filler"])
def test_filler_image_keeps_fewer_than_r_rows(name):
    ref = _oracle(name)
    nk = ref["num_kept"]
    assert 0 < nk[-1] < 300 and (nk[:-1] == 300).all()
    B = len(nk)
    assert (ref["keep_idx"][(B - 1) * 300 + nk[-1]:] == -1).all()
    assert (ref["scores"][(B - 1) * 300 + nk[-1]:] == 0).all()


def test_strip_pairs_are_listed_only_with_swapped_map_bounds():
    """On the 16 x 80 FocusChip map, each strip pair is two whole-image boxes at column offset 16 / 17 of anchor type
    20.  The overlap map does not list them (offset >= H), so FastNMS keeps both; their anchors' IoU at the map's
    swapped shift is >= 0.3, so bounds checked against the wrong dimension would list them and drop one."""
    c = C.build("resnet101-focuschips-strip-pairs-flags2")
    H, W, A = c["H"], c["W"], c["A"]
    assert (H, W) == (16, 80)
    anchors = O.generate_anchors(16, c["kw"]["scales"], c["kw"]["ratios"])
    a = anchors[20].astype(np.float64)
    area = (a[2] - a[0] + 1) * (a[3] - a[1] + 1)
    pairs = C.strip_pairs(H, W)
    for _, h, w1, w2 in pairs:
        sy = (w2 - w1) * 16.0
        inter = (a[2] - a[0] + 1) * max(0.0, a[3] - a[1] + 1 - sy)
        assert w2 - w1 >= H and inter / (2 * area - inter) >= 0.3
    for flags in (2, 3):
        ref = _oracle("resnet101-focuschips-strip-pairs-flags%d" % flags)
        for b in range(len(c["im_info"])):
            kept = set(ref["keep_idx"][b * 300:(b + 1) * 300].tolist())
            for t, h, w1, w2 in pairs:
                assert {t * H * W + h * W + w1, t * H * W + h * W + w2} <= kept


def test_tied_pairs():
    cls_prob, bbox_pred, im_info, (i, j) = C.tied_pair(overlap=False)
    ref = O.multi_proposal(cls_prob, bbox_pred, im_info, libm_exp=False)
    assert list(ref["keep_idx"][:2]) == [1, 32] == [i, j]
    assert cls_prob[0, 21:].ravel()[i] == cls_prob[0, 21:].ravel()[j]
    # disjoint boxes: the order is decided by the tie rule alone
    b1, b2 = ref["rois"][0, 1:], ref["rois"][1, 1:]
    assert b1[3] < b2[1] or b2[3] < b1[1] or b1[2] < b2[0] or b2[2] < b1[0]
    cls_prob, bbox_pred, im_info, (i, j) = C.tied_pair(overlap=True)
    ref = O.multi_proposal(cls_prob, bbox_pred, im_info, libm_exp=False)
    assert ref["keep_idx"][0] == i == 5 and j == 1026 and j not in ref["keep_idx"]
    assert (ref["rois"][0, 1:] == [0, 0, 255, 255]).all()
