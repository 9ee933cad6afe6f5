"""CPU checks that pin the oracle itself (no GPU, no product code)."""
import ctypes
import os
import sys

import numpy as np
import pytest

import oracle_lib as O
from sniper_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_expf_is_correctly_rounded():
    """oracle_expf == round_to_float(exp in double) exactly, and within 1 ulp of glibc expf
    (glibc's expf is documented <0.502 ulp, i.e. not always correctly rounded)."""
    libm = ctypes.CDLL("libm.so.6")
    libm.expf.restype = ctypes.c_float
    libm.expf.argtypes = [ctypes.c_float]
    rng = np.random.RandomState(0)
    xs = np.concatenate([rng.randn(40000) * 0.5, rng.uniform(-20, 20, 10000), [0.0, -0.0, 1.0, -1.0, 88.0, -100.0]])
    xs = xs.astype(np.float32)
    mine = np.array([O.lib().oracle_expf(float(x)) for x in xs], np.float32)
    ref = np.exp(xs.astype(np.float64)).astype(np.float32)
    np.testing.assert_array_equal(mine, ref)
    glibc = np.array([libm.expf(float(x)) for x in xs[:5000]], np.float32)
    assert np.all(np.abs(mine[:5000] - glibc) <= np.abs(glibc) * 1.2e-7)
    assert O.lib().oracle_expf(200.0) == np.inf and O.lib().oracle_expf(-200.0) == 0.0


def test_anchors_match_numpy_generate_anchors():
    # independent restatement of lib/data_utils/generate_anchor.py:8-77 semantics for these ratios/scales
    a = O.generate_anchors(16, synth.SCALES_RES101, synth.RATIOS)
    assert a.shape == (21, 4)
    # ratio 1, scale 2 -> 32x32 box centred at 7.5
    np.testing.assert_array_equal(a[7], np.array([-8.0, -8.0, 23.0, 23.0], np.float32))
    # widths/heights: ratio 0.5 -> w=23*s,h=12*s ; ratio 2 -> w=11*s,h=22*s (cu:89-98)
    w = a[:, 2] - a[:, 0] + 1
    h = a[:, 3] - a[:, 1] + 1
    s = np.array(synth.SCALES_RES101, np.float32)
    np.testing.assert_array_equal(w[:7], 23 * s)
    np.testing.assert_array_equal(h[:7], 12 * s)
    np.testing.assert_array_equal(w[14:], 11 * s)
    np.testing.assert_array_equal(h[14:], 22 * s)


def _np_decode(cls_prob, bbox_pred, im_info, vr, anchors, stride):
    """Independent vectorised numpy restatement of getProps (multi_proposal_target.cu:263-331) in float64 geometry."""
    B, A4, H, W = bbox_pred.shape
    A = A4 // 4
    sx = (np.arange(W) * stride).astype(np.float32)
    sy = (np.arange(H) * stride).astype(np.float32)
    out = np.zeros((B, A, H, W, 6), np.float32)
    for b in range(B):
        for a in range(A):
            x1 = anchors[a, 0] + sx[None, :] + np.zeros((H, 1), np.float32)
            y1 = anchors[a, 1] + sy[:, None] + np.zeros((1, W), np.float32)
            x2 = anchors[a, 2] + sx[None, :] + np.zeros((H, 1), np.float32)
            y2 = anchors[a, 3] + sy[:, None] + np.zeros((1, W), np.float32)
            score = cls_prob[b, A + a].copy()
            width = (x2 - x1).astype(np.float64) + 1.0
            height = (y2 - y1).astype(np.float64) + 1.0
            width = width.astype(np.float32)
            height = height.astype(np.float32)
            cx = (x1.astype(np.float64) + 0.5 * (width.astype(np.float64) - 1.0)).astype(np.float32)
            cy = (y1.astype(np.float64) + 0.5 * (height.astype(np.float64) - 1.0)).astype(np.float32)
            dx, dy, dw, dh = bbox_pred[b, 4 * a], bbox_pred[b, 4 * a + 1], bbox_pred[b, 4 * a + 2], bbox_pred[b, 4 * a + 3]
            pcx = (dx * width).astype(np.float32) + cx
            pcy = (dy * height).astype(np.float32) + cy
            pw = np.exp(dw.astype(np.float64)).astype(np.float32) * width
            ph = np.exp(dh.astype(np.float64)).astype(np.float32) * height
            px1 = (pcx.astype(np.float64) - 0.5 * (pw.astype(np.float64) - 1.0)).astype(np.float32)
            py1 = (pcy.astype(np.float64) - 0.5 * (ph.astype(np.float64) - 1.0)).astype(np.float32)
            px2 = (pcx.astype(np.float64) + 0.5 * (pw.astype(np.float64) - 1.0)).astype(np.float32)
            py2 = (pcy.astype(np.float64) + 0.5 * (ph.astype(np.float64) - 1.0)).astype(np.float32)
            iw, ih = np.float32(im_info[b, 1] - np.float32(1)), np.float32(im_info[b, 0] - np.float32(1))
            px1 = np.maximum(np.minimum(px1, iw), np.float32(0))
            py1 = np.maximum(np.minimum(py1, ih), np.float32(0))
            px2 = np.maximum(np.minimum(px2, iw), np.float32(0))
            py2 = np.maximum(np.minimum(py2, ih), np.float32(0))
            small = ((py2 - py1) < 3) & ((px2 - px1) < 3)
            px1 = np.where(small, px1 - 1, px1)
            py1 = np.where(small, py1 - 1, py1)
            px2 = np.where(small, px2 + 1, px2)
            py2 = np.where(small, py2 + 1, py2)
            score = np.where(small, np.float32(-1), score)
            area = (px2 - px1) * (py2 - py1)
            bad = (area >= vr[b, 1] * vr[b, 1]) | (area < vr[b, 0] * vr[b, 0])
            score = np.where(bad, np.float32(-1), score)
            out[b, a] = np.stack([px1, py1, px2, py2, score, area], -1)
    return out.reshape(-1, 6)


def _np_greedy_nms(dets, post, thresh=0.7):
    """Independent restatement of NonMaximumSuppression for tie-free scores: sort + greedy."""
    order = np.argsort(-dets[:, 4], kind="stable")
    alive = dets[:, 4] != -1
    keep = []
    for i in order:
        if not alive[i]:
            continue
        if len(keep) == post:
            break
        keep.append(i)
        xx1 = np.maximum(dets[i, 0], dets[:, 0])
        yy1 = np.maximum(dets[i, 1], dets[:, 1])
        xx2 = np.minimum(dets[i, 2], dets[:, 2])
        yy2 = np.minimum(dets[i, 3], dets[:, 3])
        w = np.maximum(np.float32(0), xx2 - xx1 + np.float32(1))
        h = np.maximum(np.float32(0), yy2 - yy1 + np.float32(1))
        inter = w * h
        ovr = inter / ((dets[i, 5] + dets[:, 5]) - inter)
        alive &= ~(ovr > 0.7)
        alive[i] = False
    return keep


@pytest.mark.parametrize("seed,B", [(1, 2), (2, 3)])
def test_oracle_mpt_against_independent_numpy(seed, B):
    A, H, W = 21, 16, 16
    cls_prob, bbox_pred, im_info, gts, vr = synth.mpt_inputs(seed, B, A, H, W)
    res = O.multi_proposal_target(cls_prob, bbox_pred, im_info, gts, vr, post=300)
    anchors = O.generate_anchors(16, synth.SCALES_RES101, synth.RATIOS)
    dets = _np_decode(cls_prob, bbox_pred, im_info, vr, anchors, 16)
    # decode: numpy's exp is libm double exp -> identical except at ~1e-7 of inputs
    assert np.mean(dets != res["dets"]) < 1e-5
    n = A * H * W
    for b in range(B):
        d = res["dets"][b * n:(b + 1) * n]
        valid_scores = d[d[:, 4] != -1, 4]
        if len(np.unique(valid_scores)) != len(valid_scores):
            continue  # tie order is only defined by the sequential emulation
        keep = _np_greedy_nms(d, 300)
        nk = res["num_kept"][b]
        assert nk == len(keep)
        np.testing.assert_array_equal(res["keep_idx"][b * 300:b * 300 + nk], np.array(keep, np.int32))
    # structure of the outputs
    rois = res["rois"].reshape(B, 300, 5)
    for b in range(B):
        assert np.all(rois[b, :, 0] == b)
        numgt = int((gts[b, :, 4] != -1).sum())
        for j in range(numgt):
            g = gts[b, j]
            a = (g[2] - g[0]) * (g[3] - g[1])
            if vr[b, 0] ** 2 <= a <= vr[b, 1] ** 2:
                np.testing.assert_array_equal(rois[b, 300 - numgt + j, 1:], g[:4])
                assert res["label"][b * 300 + 300 - numgt + j] == g[4]  # IoU(gt,gt)=1 > 0.5 unless a better gt... first-max
    lab = res["label"]
    w = res["bbox_weight"]
    assert np.all((w == 0) | (w == 1))
    assert np.all((lab > 0) == (w[:, 0] == 1))
    assert np.all(res["bbox_target"][w[:, 0] == 0] == 1.0)


def test_oracle_psroi_backward_is_gradient_of_forward():
    # shapes of the reference's own numeric-gradient test (test_operator.py:4358-4389)
    rng = np.random.RandomState(3)
    data = rng.rand(1, 18, 14, 14).astype(np.float32)
    rois = np.array([[0, 10, 22, 161, 173], [0, 20, 15, 154, 160]], np.float32)
    trans = (rng.rand(2, 4, 3, 3).astype(np.float32) - 0.5)
    kw = dict(spatial_scale=0.0625, output_dim=2, group_size=3, pooled=3, part_size=3, spp=4, trans_std=0.1)
    out, cnt, _ = O.deform_psroi_fwd(data, rois, trans, no_trans=False, **kw)
    g = rng.randn(*out.shape).astype(np.float32)
    dd, td = O.deform_psroi_bwd(g, cnt, data, rois, trans, no_trans=False, **kw)
    eps = 1e-2
    for _ in range(20):
        idx = tuple(rng.randint(0, s) for s in data.shape)
        dp, dm = data.copy(), data.copy()
        dp[idx] += eps
        dm[idx] -= eps
        num = ((O.deform_psroi_fwd(dp, rois, trans, no_trans=False, **kw)[0].astype(np.float64) -
                O.deform_psroi_fwd(dm, rois, trans, no_trans=False, **kw)[0]) * g).sum() / (2 * eps)
        assert abs(num - dd[idx]) <= 2e-3 + 2e-2 * abs(num)
    # plain PSROI
    o2, bins = O.psroi_fwd(data, rois, 0.0625, 2, 3, 3)
    g2 = rng.randn(*o2.shape).astype(np.float32)
    d2 = O.psroi_bwd(g2, rois, data.shape, 0.0625, 2, 3, 3)
    for _ in range(20):
        idx = tuple(rng.randint(0, s) for s in data.shape)
        dp, dm = data.copy(), data.copy()
        dp[idx] += eps
        dm[idx] -= eps
        num = ((O.psroi_fwd(dp, rois, 0.0625, 2, 3, 3)[0].astype(np.float64) - O.psroi_fwd(dm, rois, 0.0625, 2, 3, 3)[0]) * g2).sum() / (2 * eps)
        assert abs(num - d2[idx]) <= 2e-3 + 2e-2 * abs(num)


def test_oracle_cpu_nms_vs_numpy():
    rng = np.random.RandomState(2)
    rois = synth.rois_for_pool(rng, 600, 1)
    dets = np.concatenate([rois[:, 1:], rng.rand(600, 1).astype(np.float32)], 1).astype(np.float32)
    keep = O.cpu_nms(dets, 0.7)
    # independent numpy restatement of lib/nms/nms.py:90-127 (py nms, same >= ... well '>' there) with '>=' rule
    x1, y1, x2, y2, sc = dets.T
    areas = (x2 - x1 + 1) * (y2 - y1 + 1)
    order = sc.argsort()[::-1]
    kp = []
    while order.size > 0:
        i = order[0]
        kp.append(i)
        xx1 = np.maximum(x1[i], x1[order[1:]]); yy1 = np.maximum(y1[i], y1[order[1:]])
        xx2 = np.minimum(x2[i], x2[order[1:]]); yy2 = np.minimum(y2[i], y2[order[1:]])
        w = np.maximum(np.float32(0.0), xx2 - xx1 + 1); h = np.maximum(np.float32(0.0), yy2 - yy1 + 1)
        inter = w * h
        ovr = inter / (areas[i] + areas[order[1:]] - inter)
        order = order[np.where(~(ovr >= 0.7))[0] + 1]
    np.testing.assert_array_equal(keep, np.array(kp, np.int32))
    # soft-nms: scores decay, survivors above threshold, count <= N
    out = O.cpu_soft_nms(dets, sigma=0.55)
    assert 0 < out.shape[0] <= 600 and np.all(out[:, 4] >= 0.001)
    assert abs(out[0, 4] - dets[:, 4].max()) < 1e-7


def test_bbox_overlaps_oracle():
    rng = np.random.RandomState(5)
    a = synth.rois_for_pool(rng, 50, 1)[:, 1:].astype(np.float64)
    b = synth.rois_for_pool(rng, 30, 1)[:, 1:].astype(np.float64)
    ov = O.bbox_overlaps(a, b)
    # restatement of bbox_overlaps_py (lib/bbox/bbox_transform.py:12-32)
    for k in range(30):
        ba = (b[k, 2] - b[k, 0] + 1) * (b[k, 3] - b[k, 1] + 1)
        for n in range(50):
            iw = min(a[n, 2], b[k, 2]) - max(a[n, 0], b[k, 0]) + 1
            ih = min(a[n, 3], b[k, 3]) - max(a[n, 1], b[k, 1]) + 1
            e = 0.0
            if iw > 0 and ih > 0:
                e = iw * ih / ((a[n, 2] - a[n, 0] + 1) * (a[n, 3] - a[n, 1] + 1) + ba - iw * ih)
            assert ov[n, k] == e


# ---------------------------------------------------------------------------------------------------------------
# Pinning against the REFERENCE ITSELF: MultiProposalTargetOp<cpu> / MultiProposalGPUOp<cpu> compiled from
# /root/reference/SNIPER-mxnet/src/operator/{multi_proposal_target,multi_proposal}.cc into oracle/_ref (oracle/Makefile).
# ---------------------------------------------------------------------------------------------------------------
def _tie_free(cls_prob, seed):
    """Replaces the foreground scores by a random permutation of distinct values in (0, 1)."""
    B, A2, H, W = cls_prob.shape
    A = A2 // 2
    n = B * A * H * W
    rng = np.random.RandomState(1000 + seed)
    fg = ((rng.permutation(n) + 1.0) / (n + 1.0)).astype(np.float32).reshape(B, A, H, W)
    assert len(np.unique(fg)) == n
    out = cls_prob.copy()
    out[:, A:] = fg
    out[:, :A] = 1.0 - fg
    return out


def _need_ref(x):
    if x is None:
        pytest.skip("oracle/_ref reference operator binary not built (needs /root/reference at build time)")
    return x


@pytest.mark.parametrize("seed,B,bbox_scale", [(0, 2, 1.0), (1, 3, 2.0), (5, 1, 0.5)])
def test_cpuop_restatement_is_bit_identical_to_the_reference_cpu_operator(seed, B, bbox_scale):
    """oracle/mpt_cpuop.c == the reference's own MultiProposalTargetOp<cpu>::Forward, every output, every bit
    (tie-free scores: std::sort leaves the order of equal scores unspecified)."""
    cls_prob, bbox_pred, im_info, gts, vr = synth.mpt_inputs(seed, B)
    cls_prob = _tie_free(cls_prob, seed)
    ref = _need_ref(O.ref_multi_proposal_target(cls_prob, bbox_pred, im_info, gts, vr, bbox_scale=bbox_scale))
    mine = O.multi_proposal_target_cpuop(cls_prob, bbox_pred, im_info, gts, vr, bbox_scale=bbox_scale)
    assert (mine["num_kept"] > 50).all()
    for k in ("rois", "label", "bbox_weight", "bbox_target"):
        assert mine[k].tobytes() == ref[k].tobytes(), k
    assert (ref["label"] > 0).sum() > 0 and (ref["bbox_weight"] > 0).sum() > 0


def test_gpuop_oracle_agrees_with_the_reference_cpu_operator_where_the_two_sources_agree():
    """oracle/mpt.c restates the GPU operator (.cu); the reference binary that runs here is the CPU operator (.cc).
    Where the two reference sources agree, mpt.c must reproduce the binary:
      * anchor grid + delta decode + clip: identical boxes for every anchor that neither operator filters and whose
        exp() agrees between libm expf and the correctly rounded oracle_expf (all but a handful);
      * GT append, IoU assignment, labels, weights: identical on the rois the binary produced;
      * regression targets: the .cu uses (10,10,5,5), the .cc bbox_scale*(5,5,10,10) -> columns 0,1 equal the binary
        run with bbox_scale=2, columns 2,3 the binary run with bbox_scale=0.5.
    What stays pinned by the .cu text only: min-size rule, area/range rule, +1-free IoU areas, argmax tie order,
    filler boxes (DESIGN.md section 4)."""
    B = 2
    cls_prob, bbox_pred, im_info, gts, vr = synth.mpt_inputs(3, B)
    cls_prob = _tie_free(cls_prob, 3)
    wide = np.tile(np.array([[0.0, 1e4]], np.float32), (B, 1))           # no valid-range filtering in either operator
    ref2 = _need_ref(O.ref_multi_proposal_target(cls_prob, bbox_pred, im_info, gts, wide, bbox_scale=2.0))
    ref05 = O.ref_multi_proposal_target(cls_prob, bbox_pred, im_info, gts, wide, bbox_scale=0.5)
    cpu = O.multi_proposal_target_cpuop(cls_prob, bbox_pred, im_info, gts, wide, bbox_scale=2.0)
    gpu = O.multi_proposal_target(cls_prob, bbox_pred, im_info, gts, wide)
    assert cpu["rois"].tobytes() == ref2["rois"].tobytes()               # so cpu["dets"] are the binary's decoded rows
    # ---- decode
    dc, dg = cpu["dets"], gpu["dets"]
    unfiltered = (dc[:, 4] != -1) & (dg[:, 4] != -1)
    same = (dc[:, :4] == dg[:, :4]).all(1)
    assert unfiltered.mean() > 0.9
    assert (same | ~unfiltered).mean() > 0.999                           # the rest: expf vs correctly rounded exp
    dwh = bbox_pred.reshape(B, 21, 4, 32, 32)[:, :, 2:].transpose(0, 1, 3, 4, 2).reshape(-1, 2)
    import ctypes
    libm = ctypes.CDLL("libm.so.6")
    libm.expf.restype = ctypes.c_float
    libm.expf.argtypes = [ctypes.c_float]
    flat = dwh.astype(np.float32).ravel()
    e_libm = np.array([libm.expf(float(v)) for v in flat], np.float32)       # what the reference binary calls
    e_cr = np.array([O.lib().oracle_expf(float(v)) for v in flat], np.float32)   # what mpt.c / the CUDA kernel use
    exp_agrees = (e_libm == e_cr).reshape(-1, 2).all(1)
    assert exp_agrees.mean() > 0.99
    assert (same | ~unfiltered | ~exp_agrees).all()
    # ---- assignment on the binary's rois (GT rows already appended; appending again is idempotent)
    R = 300
    rois = ref2["rois"].copy()
    label = np.zeros(B * R, np.float32)
    bt = np.zeros((B * R, 4), np.float32)
    bw = np.zeros((B * R, 4), np.float32)
    O.lib().oracle_assign_targets(O._p(rois), O._p(O.f32(gts)), O._p(wide), O.I(B), O.I(R), O.I(100), O._p(label),
                                  O._p(bt), O._p(bw))
    assert rois.tobytes() == ref2["rois"].tobytes()
    assert label.tobytes() == ref2["label"].tobytes() and bw.tobytes() == ref2["bbox_weight"].tobytes()
    pos = bw[:, 0] > 0
    assert pos.sum() > 10
    assert bt[:, :2].tobytes() == ref2["bbox_target"][:, :2].tobytes()
    assert bt[:, 2:].tobytes() == ref05["bbox_target"][:, 2:].tobytes()


def test_reference_inference_operator_runs():
    """MultiProposalGPUOp<cpu> (multi_proposal.cc) from the reference binary: kept rows are sorted by score, clipped to
    the image and mutually below the NMS threshold (smoke check of the harness used by the inference-path oracle)."""
    B = 1
    cls_prob, bbox_pred, im_info, gts, vr = synth.mpt_inputs(2, B)
    cls_prob = _tie_free(cls_prob, 2)
    out = _need_ref(O.ref_multi_proposal(cls_prob, bbox_pred, im_info))
    rois, scores = out
    k = int((scores > 0).sum())
    assert k > 50 and (np.diff(scores[:k]) <= 0).all()
    assert (rois[:k, 1:] >= 0).all() and (rois[:k, [1, 3]] <= im_info[0, 1] - 1).all()


@pytest.mark.parametrize("seed,B,HW", [(11, 1, 32), (12, 2, 32), (13, 1, 20)])
def test_inference_op_restatement_is_bit_identical_to_the_reference_cpu_operator(seed, B, HW):
    """oracle/mp_cpuop.c (flags = 0, libm exp) == MultiProposalGPUOp<cpu>::Forward of the reference binary on the kept
    rows (boxes and scores); the rows after them are rand() fillers in the reference.  HW=20: 8400 anchors < 12000."""
    cls_prob, bbox_pred, im_info, gts, vr = synth.mpt_inputs(seed, B, 21, HW, HW)
    cls_prob = _tie_free(cls_prob, seed)
    rois, scores = _need_ref(O.ref_multi_proposal(cls_prob, bbox_pred, im_info))
    mine = O.multi_proposal(cls_prob, bbox_pred, im_info, libm_exp=True)
    for b in range(B):
        k = int(mine["num_kept"][b])
        assert k > 50
        sl = slice(b * 300, b * 300 + k)
        assert mine["rois"][sl].tobytes() == rois[sl].tobytes()
        assert mine["scores"][sl].tobytes() == scores[sl].tobytes()
        assert (scores[b * 300 + k:(b + 1) * 300] == 0).all()       # the reference's filler rows carry score 0


@pytest.mark.parametrize("name", ["resnet101-s0-landscape", "resnet101-s0-portrait", "resnet101-largest-tie_free",
                                  "mobilenetv2-s0-landscape", "mobilenetv2-s0-portrait"])
def test_inference_op_restatement_matches_the_reference_at_tester_canvases(name):
    """The same pin at the Tester's canvases (tests/multi_proposal_cases.py, tie-free scores): rectangular maps in both
    orientations, several images with their own im_info smaller than the canvas, the ResNet-101 anchors at stride 16
    (up to 225792 anchors per image) and the MobileNetV2 anchors at stride 32 with 6000 pre-NMS rows.  The reference
    operator always sorts min(12000, A*H*W) rows (multi_proposal.cc:176); the 6000-row cases are compared where that
    cannot matter, which the oracle itself shows: its 300 rows are the same with 6000 and with 12000."""
    import multi_proposal_cases as C
    c = C.build(name)
    assert c["regime"] == "tie_free" and c["flags"] == 0
    cls_prob, bbox_pred, im_info, pre = c["cls_prob"], c["bbox_pred"], c["im_info"], c["pre"]
    rois, scores = _need_ref(O.ref_multi_proposal(cls_prob, bbox_pred, im_info, pre=pre, **c["kw"]))
    mine = O.multi_proposal(cls_prob, bbox_pred, im_info, pre=pre, libm_exp=True, **c["kw"])
    if pre < 12000:
        wide = O.multi_proposal(cls_prob, bbox_pred, im_info, pre=12000, libm_exp=True, **c["kw"])
        assert all(mine[k].tobytes() == wide[k].tobytes() for k in ("rois", "scores", "keep_idx"))
    B = len(im_info)
    assert B >= 2 and c["H"] != c["W"] and (im_info[:, 0] != im_info[:, 1]).all()
    for b in range(B):
        k = int(mine["num_kept"][b])
        assert k > 50
        sl = slice(b * 300, b * 300 + k)
        assert mine["rois"][sl].tobytes() == rois[sl].tobytes(), b
        assert mine["scores"][sl].tobytes() == scores[sl].tobytes(), b
        assert (scores[b * 300 + k:(b + 1) * 300] == 0).all()
        assert (rois[sl, 3] <= im_info[b, 1] - 1).all() and (rois[sl, 4] <= im_info[b, 0] - 1).all()


def test_inference_op_gpu_build_extras():
    """The two extras of multi_proposal.cu (pinned by the .cu text only): anchor-type suppression removes exactly the
    anchor types (i+4)%7==0 / (i+2)%7==0 from the output; FastNMS keeps a superset-or-equal of rows early in the list
    (it tests fewer pairs) and is identical to the plain NMS when the overlap map admits every pair (thresh <= 0)."""
    cls_prob, bbox_pred, im_info, gts, vr = synth.mpt_inputs(21, 1)
    cls_prob = _tie_free(cls_prob, 21)
    plain = O.multi_proposal(cls_prob, bbox_pred, im_info)
    sup = O.multi_proposal(cls_prob, bbox_pred, im_info, flags=1)
    types = sup["keep_idx"][:int(sup["num_kept"][0])] // (32 * 32)
    assert not np.isin(types % 7, [3, 5]).any()
    assert np.isin(plain["keep_idx"][:300] // 1024 % 7, [3, 5]).any()
    fast_all = O.multi_proposal(cls_prob, bbox_pred, im_info, flags=2, roi_iou_thresh=-1.0)
    assert fast_all["rois"].tobytes() == plain["rois"].tobytes()
    fast = O.multi_proposal(cls_prob, bbox_pred, im_info, flags=2, roi_iou_thresh=0.3)
    assert fast["keep_idx"][0] == plain["keep_idx"][0] and int(fast["num_kept"][0]) == 300


@pytest.mark.parametrize("seed,n_gt,n_valid", [(0, 12, 9), (1, 30, 30), (2, 5, 2), (3, 1, 0), (4, 60, 41)])
def test_anchor_target_oracle_matches_the_reference_anchor_worker(seed, n_gt, n_valid):
    """oracle/anchor_target_np.py == the reference's own anchor_worker.worker (data_workers.py:130-371, executed here by
    oracle/run_ref_anchor_worker.py with its own generate_anchors / bbox_transform / Cython bbox_overlaps): labels after
    the reference's npr.choice subsampling, positive-anchor indices and their regression targets, bit for bit."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import anchor_target_np as AT
    try:
        import run_ref_anchor_worker as R
        worker = R.load_reference_worker()(R.make_cfg(), 512)
    except (ImportError, OSError) as e:
        pytest.skip("reference anchor_worker not runnable here: %s" % e)
    boxes, classes, gtids, nids = R.synth_case(seed, n_gt, n_valid)
    lab_ref, tg_ref, pids_ref, fgt = R.run_reference(worker, boxes, classes, gtids, nids, seed=100 + seed)
    valid = np.zeros(n_gt, bool)
    valid[nids] = True
    for i in range(n_gt):                         # a GT identical to a valid one counts as valid (mov == 1, :262-272)
        if not valid[i] and n_valid and (boxes[nids] == boxes[i]).all(1).any():
            valid[i] = True
    res = AT.anchor_target(boxes[valid], boxes[~valid], np.array([512, 512, 1.0]))
    disable = AT.subsample(res["labels"], np.random.RandomState(100 + seed))
    labels = res["labels"].copy()
    labels[disable] = -1
    lab, tg, w = AT.pack(labels, res["targets"], 32, 32, res["A"])
    assert lab.tobytes() == lab_ref.tobytes()
    pids = np.stack(np.where(w == 1))
    assert np.array_equal(pids, pids_ref)
    assert tg[tuple(pids)].tobytes() == tg_ref.tobytes()
    assert (lab_ref == 1).sum() <= 128 and (lab_ref >= 0).sum() <= 256
    assert np.array_equal(fgt[:n_gt, :4], boxes) and (fgt[n_gt:] == -1).all()


@pytest.mark.parametrize("case", ["no_gt", "hundred_gt", "everything_filtered", "B17", "tiny_boxes"])
def test_cpuop_restatement_edge_cases_against_the_reference_binary(case):
    """Edge cases of the reference CPU operator reproduced bit for bit: no ground truth, all 100 GT slots used, a valid
    range that filters every proposal (only filler rows + GT rows remain), B = 17 (> the 16 images the reference's GPU
    operator sizes its host buffers for), deltas that shrink every box below the min-size test."""
    B = 17 if case == "B17" else 2
    cls_prob, bbox_pred, im_info, gts, vr = synth.mpt_inputs(40, B)
    cls_prob = _tie_free(cls_prob, 40)
    if case == "no_gt":
        gts = np.full_like(gts, -1.0)
    elif case == "hundred_gt":
        rng = np.random.RandomState(9)
        x1 = rng.uniform(0, 400, (B, 100)); y1 = rng.uniform(0, 400, (B, 100))
        gts = np.stack([x1, y1, x1 + rng.uniform(20, 100, (B, 100)), y1 + rng.uniform(20, 100, (B, 100)),
                        rng.randint(1, 81, (B, 100)).astype(np.float64)], 2).astype(np.float32)
    elif case == "everything_filtered":
        vr = np.tile(np.array([[600.0, 601.0]], np.float32), (B, 1))
    elif case == "tiny_boxes":
        bbox_pred = bbox_pred.copy()
        bbox_pred.reshape(B, 21, 4, 32, 32)[:, :, 2:] = -8.0          # exp(-8) * anchor size < 3 px
    ref = _need_ref(O.ref_multi_proposal_target(cls_prob, bbox_pred, im_info, gts, vr))
    mine = O.multi_proposal_target_cpuop(cls_prob, bbox_pred, im_info, gts, vr)
    for k in ("rois", "label", "bbox_weight", "bbox_target"):
        assert mine[k].tobytes() == ref[k].tobytes(), (case, k)
    if case in ("everything_filtered", "tiny_boxes"):
        assert (mine["num_kept"] == 0).all() and (ref["rois"][0, 1:] == [0, 0, 100, 100]).all()
    if case == "hundred_gt":
        assert (ref["label"] > 0).sum() > 50          # GT rows inside the valid range are appended and match themselves
