"""Tensor-level wrappers over the C-ABI (torch tensors are only device memory + streams here).

Every function launches on torch's current CUDA stream, allocates outputs with torch, and raises
`SniperError` when the native call fails.  There is no CPU fallback.
"""
import ctypes
import os

import numpy as np
import torch

from . import _lib as _libmod
from ._lib import check, lib

TF32, BF16 = 0, 1
NCHW, NHWC = 0, 1


def reset_launch_count():
    _libmod.launches[0] = 0


def launch_count():
    """GPU kernels launched through the C-ABI since the last reset."""
    return _libmod.launches[0]


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _f32(t):
    assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), "expected contiguous fp32 CUDA tensor"
    return t


def _farr(v):
    a = np.ascontiguousarray(np.asarray(v, dtype=np.float32))
    return a, a.ctypes.data_as(ctypes.c_void_p)


def _iarr(v):
    a = np.ascontiguousarray(np.asarray(v, dtype=np.int32))
    return a, a.ctypes.data_as(ctypes.c_void_p)


def generate_anchors(feat_stride, scales, ratios):
    """multi_proposal_target.cu:75-114 anchor table, [len(ratios)*len(scales), 4] (ratio-major)."""
    s, sp = _farr(scales)
    r, rp = _farr(ratios)
    out = np.zeros((len(r) * len(s), 4), np.float32)
    check(lib().sniper_generate_anchors(int(feat_stride), sp, len(s), rp, len(r), out.ctypes.data_as(ctypes.c_void_p)))
    return out


def multi_proposal(cls_prob, bbox_pred, im_info, *, feat_stride=16, scales=(2, 4, 7, 10, 13, 16, 24),
                   ratios=(0.5, 1, 2), rpn_pre_nms_top_n=12000, rpn_post_nms_top_n=300, threshold=0.7,
                   suppress_anchor_types=False, fast_nms=False, roi_iou_thresh=0.3, layout=NCHW, return_keep=False,
                   return_fallback=False):
    """MultiProposal forward -- the inference proposal operator (multi_proposal.cc:273-374 semantics: decode, min-size
    filter, the rpn_pre_nms_top_n best anchors, greedy NMS), on device; suppress_anchor_types / fast_nms select the two
    extras of the reference's GPU build (multi_proposal.cu:505-508, 267-387).  Returns rois [B*R,5], scores [B*R]
    (+ keep_idx [B*R] original anchor indices / -1 for filler rows, num_kept [B]; + the per-image flag of the bit-mask
    NMS, 1 = the sequential kernel ran, meaningful unless SNIPER_NMS_FAST=0).

    Equal scores are taken in ascending anchor index, by the pre-NMS selection and by the NMS: the rule of the oracle
    (oracle/mp_cpuop.c), since the reference sorts with std::sort, whose order of equal scores is unspecified.  The
    training operator, multi_proposal_target, breaks NMS ties in the reference GPU kernel's scan order instead."""
    _f32(cls_prob), _f32(bbox_pred), _f32(im_info)
    A = len(scales) * len(ratios)
    if layout == NCHW:
        B, H, W = bbox_pred.shape[0], bbox_pred.shape[2], bbox_pred.shape[3]
        assert bbox_pred.shape[1] == 4 * A and cls_prob.numel() == B * 2 * A * H * W
        sc, dc = 0, 0
    else:
        B, H, W = bbox_pred.shape[0], bbox_pred.shape[1], bbox_pred.shape[2]
        sc, dc = cls_prob.shape[3], bbox_pred.shape[3]
        assert dc >= 4 * A and sc >= 2 * A
    R = int(rpn_post_nms_top_n)
    dev = cls_prob.device
    rois = torch.empty(B * R, 5, device=dev)
    scores = torch.empty(B * R, device=dev)
    keep = torch.empty(B * R, dtype=torch.int32, device=dev) if return_keep else None
    nkept = torch.empty(B, dtype=torch.int32, device=dev) if return_keep else None
    L = lib()
    ws_bytes = L.sniper_multi_proposal_workspace_bytes(B, A, H, W, int(rpn_pre_nms_top_n))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    s, sp = _farr(scales)
    r, rp = _farr(ratios)
    check(L.sniper_multi_proposal_fwd(
        _ptr(cls_prob), _ptr(bbox_pred), _ptr(im_info), B, A, H, W, int(rpn_pre_nms_top_n), R, int(feat_stride), sp,
        len(s), rp, len(r), float(threshold), (1 if suppress_anchor_types else 0) | (2 if fast_nms else 0),
        float(roi_iou_thresh), layout, sc, dc, _ptr(rois),
        _ptr(scores), _ptr(keep), _ptr(nkept), _ptr(ws), ws_bytes, _stream()))
    if return_fallback:
        # per-image flag written by mpt_nms_fast_kernel after the workspace's decoded and compacted rows (16-byte
        # aligned arrays, sniper_multi_proposal_fwd)
        r16 = lambda n: (n + 15) // 16 * 16
        total, K = B * A * H * W, B * min(int(rpn_pre_nms_top_n), A * H * W)
        off = 16 * total + 2 * r16(4 * total) + 16 * K + 3 * r16(4 * K)
        fb = ws[off:off + B * 1026 * 4].view(torch.int32)[B * 1025:B * 1026].clone()
        return rois, scores, keep, nkept, fb
    if return_keep:
        return rois, scores, keep, nkept
    return rois, scores


def multi_proposal_target(cls_prob, bbox_pred, im_info, gt_boxes, valid_ranges, *, feat_stride=16,
                          scales=(2, 4, 7, 10, 13, 16, 24), ratios=(0.5, 1, 2), rpn_post_nms_top_n=300,
                          threshold=0.7, layout=NCHW, return_keep=False, return_fallback=False):
    """MultiProposalTarget forward (reference GPU-operator semantics, multi_proposal_target.cu:362-589).

    NCHW: cls_prob [B,2A,H,W] (or [B,2,A*H,W]), bbox_pred [B,4A,H,W].  NHWC: [B,H,W,2A] / [B,H,W,4A].
    Returns rois [B*R,5], label [B*R], bbox_target [B*R,4], bbox_weight [B*R,4] (+ keep_idx, num_kept).
    """
    _f32(cls_prob), _f32(bbox_pred), _f32(im_info), _f32(gt_boxes), _f32(valid_ranges)
    A = len(scales) * len(ratios)
    if layout == NCHW:
        B, H, W = bbox_pred.shape[0], bbox_pred.shape[2], bbox_pred.shape[3]
        assert bbox_pred.shape[1] == 4 * A and cls_prob.numel() == B * 2 * A * H * W
        sc, dc = 0, 0
    else:
        B, H, W = bbox_pred.shape[0], bbox_pred.shape[1], bbox_pred.shape[2]
        sc, dc = cls_prob.shape[3], bbox_pred.shape[3]
        assert dc >= 4 * A and sc >= 2 * A
    R = int(rpn_post_nms_top_n)
    max_gt = gt_boxes.shape[1]
    dev = cls_prob.device
    rois = torch.empty(B * R, 5, device=dev)
    label = torch.empty(B * R, device=dev)
    bbox_target = torch.empty(B * R, 4, device=dev)
    bbox_weight = torch.empty(B * R, 4, device=dev)
    keep = torch.empty(B * R, dtype=torch.int32, device=dev) if return_keep else None
    nkept = torch.empty(B, dtype=torch.int32, device=dev) if return_keep else None
    L = lib()
    ws_bytes = L.sniper_multi_proposal_target_workspace_bytes(B, A, H, W)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    s, sp = _farr(scales)
    r, rp = _farr(ratios)
    check(L.sniper_multi_proposal_target_fwd(
        _ptr(cls_prob), _ptr(bbox_pred), _ptr(im_info), _ptr(gt_boxes), _ptr(valid_ranges), B, A, H, W, max_gt, R,
        int(feat_stride), sp, len(s), rp, len(r), float(threshold), layout, sc, dc, _ptr(rois), _ptr(label),
        _ptr(bbox_target), _ptr(bbox_weight), _ptr(keep), _ptr(nkept), _ptr(ws), ws_bytes, _stream()))
    if return_fallback:
        # per-chip flag written by mpt_nms_fast_kernel into the workspace tail (1 = sequential emulation was used)
        off = B * A * H * W * 24 + 64
        fb = ws[off:off + B * 1026 * 4].view(torch.int32)[B * 1025:B * 1026].clone()
        return rois, label, bbox_target, bbox_weight, keep, nkept, fb
    if return_keep:
        return rois, label, bbox_target, bbox_weight, keep, nkept
    return rois, label, bbox_target, bbox_weight


def _ps_dims(data, layout):
    if layout == NCHW:
        B, C, H, W = data.shape
    else:
        B, H, W, C = data.shape
    return B, C, H, W


def deform_psroi_fwd(data, rois, trans, *, spatial_scale, output_dim, group_size, pooled_size, part_size=0,
                     sample_per_part=1, trans_std=0.0, no_trans=False, layout=NCHW, want_count=True,
                     want_sample_idx=False):
    """DeformablePSROIPooling forward (deformable_psroi_pooling.cu:71-161)."""
    _f32(data), _f32(rois)
    _, C, H, W = _ps_dims(data, layout)
    N = rois.shape[0]
    P = pooled_size
    shape = (N, output_dim, P, P) if layout == NCHW else (N, P, P, output_dim)
    out = torch.empty(shape, device=data.device)
    cnt = torch.empty(shape, device=data.device) if want_count else None
    S = sample_per_part
    sidx = torch.empty(N * output_dim * P * P, S * S, 4, dtype=torch.int32, device=data.device) if want_sample_idx else None
    ncls = 1 if no_trans else trans.shape[1] // 2
    check(lib().sniper_deform_psroi_fwd(_ptr(data), _ptr(rois), _ptr(None if no_trans else _f32(trans)), N, C, H, W,
                                        float(spatial_scale), output_dim, group_size, P, part_size, S,
                                        float(trans_std), int(no_trans), ncls, layout, _ptr(out), _ptr(cnt),
                                        _ptr(sidx), _stream()))
    return out, cnt, sidx


def deform_psroi_bwd(top_diff, data, rois, trans, *, spatial_scale, output_dim, group_size, pooled_size,
                     part_size=0, sample_per_part=1, trans_std=0.0, no_trans=False, layout=NCHW,
                     data_diff=None, trans_diff=None):
    """DeformablePSROIPooling backward (deformable_psroi_pooling.cu:203-330); returns (data_diff, trans_diff)."""
    _f32(top_diff), _f32(data), _f32(rois)
    B, C, H, W = _ps_dims(data, layout)
    N = rois.shape[0]
    if data_diff is None:
        data_diff = torch.zeros_like(data)
    if trans_diff is None and not no_trans:
        trans_diff = torch.zeros_like(trans)
    ncls = 1 if no_trans else trans.shape[1] // 2
    # product path (NHWC, one class, the channel counts of the warp-per-bin kernels, 16-byte aligned buffers): the
    # scattered contributions are summed in an fp64 scratch, which makes the gradients reproducible run to run
    if (layout == NHWC and group_size == 1 and ncls == 1 and sample_per_part <= 4 and C in (128, 256, 512)
            and all(t.data_ptr() % 16 == 0 for t in (data, data_diff, top_diff))):
        P = part_size if part_size else pooled_size
        n_acc = data_diff.numel() + (0 if no_trans else N * 2 * P * P)
        acc = torch.zeros(n_acc, dtype=torch.float64, device=data.device)
        rc = lib().sniper_deform_psroi_bwd_fp64acc(_ptr(top_diff), _ptr(data), _ptr(rois), _ptr(None if no_trans else trans),
                                                   N, B, C, H, W, float(spatial_scale), output_dim, group_size,
                                                   pooled_size, part_size, sample_per_part, float(trans_std),
                                                   int(no_trans), ncls, _ptr(data_diff), _ptr(trans_diff), _ptr(acc),
                                                   n_acc, _stream())
        if rc != -2:
            check(rc)
            if not no_trans:
                _libmod.launches[0] += 1          # + the trans_diff half of the fp64 -> fp32 step
            return data_diff, trans_diff
    check(lib().sniper_deform_psroi_bwd(_ptr(top_diff), _ptr(data), _ptr(rois), _ptr(None if no_trans else trans), N, C,
                                        H, W, float(spatial_scale), output_dim, group_size, pooled_size, part_size,
                                        sample_per_part, float(trans_std), int(no_trans), ncls, layout,
                                        _ptr(data_diff), _ptr(trans_diff), _stream()))
    return data_diff, trans_diff


def psroi_fwd(data, rois, *, spatial_scale, output_dim, group_size, pooled_size, layout=NCHW, want_bins=False):
    """PSROIPooling forward (psroi_pooling.cu:51-118)."""
    _f32(data), _f32(rois)
    B, C, H, W = _ps_dims(data, layout)
    N, P = rois.shape[0], pooled_size
    shape = (N, output_dim, P, P) if layout == NCHW else (N, P, P, output_dim)
    out = torch.empty(shape, device=data.device)
    bins = torch.empty(N * output_dim * P * P, 4, dtype=torch.int32, device=data.device) if want_bins else None
    check(lib().sniper_psroi_fwd(_ptr(data), _ptr(rois), N, C, H, W, float(spatial_scale), output_dim, group_size, P,
                                 layout, _ptr(out), _ptr(bins), _stream()))
    return out, bins


def psroi_bwd(top_diff, rois, data_shape, *, spatial_scale, output_dim, group_size, pooled_size, layout=NCHW):
    """PSROIPooling backward (psroi_pooling.cu:146-210)."""
    _f32(top_diff), _f32(rois)
    data_diff = torch.zeros(data_shape, device=top_diff.device)
    B, C, H, W = _ps_dims(data_diff, layout)
    check(lib().sniper_psroi_bwd(_ptr(top_diff), _ptr(rois), rois.shape[0], C, H, W, float(spatial_scale), output_dim,
                                 group_size, pooled_size, layout, _ptr(data_diff), _stream()))
    return data_diff


def _dt(t):
    return TF32 if t.dtype == torch.float32 else BF16


def gemm_nt(a, b, *, out=None, scale=None, bias=None, residual=None, relu=False, accumulate=False, out_dtype=None,
            stats=None):
    """C[M,N] = epi(A[M,K] @ B[N,K]^T) on wgmma tensor cores (fp32 storage -> TF32 math, or bf16 operands with fp32
    accumulation).  The output is fp32 or bf16 (default: the operands' dtype); a residual has the output's dtype."""
    assert a.is_cuda and a.dim() == 2 and b.dim() == 2 and a.shape[1] == b.shape[1] and a.dtype == b.dtype
    assert a.stride(1) == 1 and b.stride(1) == 1
    M, K = a.shape
    N = b.shape[0]
    if out is None:
        out = torch.empty(M, N, device=a.device, dtype=out_dtype or a.dtype)
    out_bf16 = out.dtype == torch.bfloat16
    assert out.shape == (M, N) and out.stride(1) == 1, "out must be [M, N] with unit column stride"
    assert residual is None or (residual.shape == (M, N) and residual.stride(1) == 1), \
        "residual must be [M, N] with unit column stride"
    assert residual is None or residual.dtype == out.dtype, "bf16 output takes a bf16 residual"
    check(lib().sniper_gemm_nt(_ptr(a), a.stride(0), _ptr(b), b.stride(0), _ptr(out), out.stride(0), M, N, K, _dt(a),
                               _ptr(scale), _ptr(bias), _ptr(residual), 0 if residual is None else residual.stride(0),
                               int(relu), int(accumulate), int(out_bf16), _ptr(stats), _stream()))
    return out


def conv_taps(kh, kw, dil, pad):
    """Tap offsets (dh, dw) in input coordinates for a kh x kw kernel, row-major over (kh, kw)."""
    dh = [i * dil - pad for i in range(kh) for _ in range(kw)]
    dw = [j * dil - pad for _ in range(kh) for j in range(kw)]
    return dh, dw


def conv2d_nhwc(x, w, *, kh, kw, stride=1, dil=1, pad=0, out=None, scale=None, bias=None, residual=None, relu=False,
                accumulate=False, taps=None, out_hw=None, out_map=None, stats=None, out_dtype=None):
    """NHWC implicit-GEMM convolution.  x: [N,H,W,Cin]; w: [Cout, kh*kw*Cin] (tap-major, channel-minor).  fp32 tensors
    run as TF32, bf16 tensors as bf16 (fp32 accumulation); the output (and the residual) may be fp32 or bf16."""
    NB, H, W, Cin = x.shape
    Cout = w.shape[0]
    dh, dw = taps if taps is not None else conv_taps(kh, kw, dil, pad)
    ntaps = len(dh)
    assert w.shape[1] == ntaps * Cin and w.is_contiguous() and x.stride(3) == 1
    x_ld = x.stride(2)
    assert x.stride(1) == W * x_ld and x.stride(0) == H * W * x_ld
    if out_hw is None:
        Ho = (H + 2 * pad - dil * (kh - 1) - 1) // stride + 1
        Wo = (W + 2 * pad - dil * (kw - 1) - 1) // stride + 1
    else:
        Ho, Wo = out_hw
    if out is None:
        out = torch.empty(NB, Ho, Wo, Cout, device=x.device, dtype=out_dtype or x.dtype)
    assert x.dtype == w.dtype and (residual is None or residual.dtype == out.dtype), "bf16 output takes a bf16 residual"
    oH, oW, os_, ooh, oow = (Ho, Wo, 1, 0, 0) if out_map is None else out_map
    _, dhp = _iarr(dh)
    _, dwp = _iarr(dw)
    check(lib().sniper_conv2d_nhwc(_ptr(x), x_ld, NB, H, W, Cin, _ptr(w), Cout, ntaps, dhp, dwp, stride, Ho, Wo,
                                   _ptr(out), _rows(out)[2], oH, oW, os_, ooh, oow, _dt(x), _ptr(scale), _ptr(bias),
                                   _ptr(residual), 0 if residual is None else _rows(residual)[2], int(relu),
                                   int(accumulate), int(out.dtype == torch.bfloat16), _ptr(stats), _stream()))
    return out


def _pixel_ld(t):
    """Row stride (elements) of an NHWC tensor whose pixels are equally spaced rows of contiguous channels."""
    assert t.dim() == 4 and t.stride(3) == 1
    NB, H, W, _ = t.shape
    ld = t.stride(2)
    assert (H == 1 or t.stride(1) == W * ld) and (NB == 1 or t.stride(0) == H * W * ld), \
        "NHWC pixel rows must be uniformly strided"
    return ld


_workspaces = {}
_replaced_workspaces = []


def _stream_workspace(copy_bytes=0):
    """The device scratch of the weight gradients on the current stream (the library never allocates): one buffer per
    (device, stream), because launches on different streams may overlap.  It holds the split-K partials and counters
    and the depthwise slab (the fixed part), then at least `copy_bytes` for the tf32 operand copies; it is grown to
    the fixed part + the next power of two when a call needs more.  Only the fixed part is zeroed, on the current
    stream (a memset node when captured), because the split-K counters must start at zero.  A replaced buffer is kept
    alive for the life of the process, because a captured CUDA graph may still hold its address."""
    idx, st = torch.cuda.current_device(), _stream()
    fixed = lib().sniper_stream_workspace_bytes()
    cur = _workspaces.get((idx, st))
    if cur is not None and cur.numel() - fixed >= copy_bytes:
        return cur
    n = fixed + (1 << (copy_bytes - 1).bit_length() if copy_bytes else 0)
    buf = torch.empty(n, dtype=torch.uint8, device=torch.device("cuda", idx))
    buf[:fixed].zero_()
    check(lib().sniper_set_stream_workspace(buf.data_ptr(), n, idx, st))
    if cur is not None:
        _replaced_workspaces.append(cur)
    _workspaces[(idx, st)] = buf
    return buf


def conv2d_wgrad_nhwc(dy, x, *, kh, kw, stride=1, dil=1, pad=0, dw_out=None, splits=8, taps=None):
    """dW[Cout, kh*kw*Cin] += dY^T * im2col(X).  dy: [N,Ho,Wo,Cout], x: [N,H,W,Cin]."""
    NB, H, W, Cin = x.shape
    _, Ho, Wo, Cout = dy.shape
    dh, dw = taps if taps is not None else conv_taps(kh, kw, dil, pad)
    ntaps = len(dh)
    assert dy.dtype == x.dtype and dy.shape[0] == NB
    dy_ld, x_ld = _pixel_ld(dy), _pixel_ld(x)
    if dw_out is None:
        dw_out = torch.zeros(Cout, ntaps * Cin, device=x.device)
    assert dw_out.dtype == torch.float32 and dw_out.is_contiguous() and dw_out.shape == (Cout, ntaps * Cin), \
        "dw_out must be a contiguous fp32 [Cout, taps * Cin]"
    _, dhp = _iarr(dh)
    _, dwp = _iarr(dw)
    _stream_workspace(lib().sniper_conv2d_wgrad_scratch_bytes(NB, H, W, Cin, Cout, ntaps, dhp, dwp, stride, Ho, Wo,
                                                               _dt(x)))
    check(lib().sniper_conv2d_wgrad_nhwc(_ptr(dy), dy_ld, _ptr(x), x_ld, NB, H, W, Cin, Cout, ntaps, dhp,
                                         dwp, stride, Ho, Wo,
                                         _ptr(dw_out), _dt(x), splits, _stream()))
    return dw_out


# ---------------------------------------------------------------------------------------------
# HBM-bound layers ([M, C] views of NHWC tensors; `ld` = row stride in elements)
# ---------------------------------------------------------------------------------------------
def _vec_aligned(t):
    """first element on a 4-channel boundary of its storage type (16 bytes fp32, 8 bytes bf16): the least any row kernel
    needs; the entry points check the rest (16 bytes for the row-blocked kernels, row strides)."""
    return t.data_ptr() % (4 * t.element_size()) == 0


def _rows(t):
    """(M, C, ld) of a tensor whose last dim is contiguous and whose leading dims collapse to rows."""
    C = t.shape[-1]
    assert t.stride(-1) == 1
    assert not t.is_cuda or _vec_aligned(t), "row kernels read whole 4-channel vectors: misaligned channel slice"
    ld = t.stride(-2) if t.dim() >= 2 else C
    M = t.numel() // C
    return M, C, ld


def _sdt(t):
    """storage dtype code of the C-ABI: 0 = fp32, 1 = bf16"""
    if t.dtype == torch.float32:
        return 0
    assert t.dtype == torch.bfloat16, "activations are fp32 or bf16"
    return 1


def affine_act(x, scale, shift, relu=True, out=None):
    M, C, ldx = _rows(x)
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=x.dtype)
    assert out.dtype == x.dtype
    check(lib().sniper_affine_act(_ptr(x), ldx, _ptr(scale), _ptr(shift), _ptr(out), _rows(out)[2], M, C, int(relu),
                                  _sdt(x), _stream()))
    return out


def cast_rows(x, dtype=None, out=None):
    """out[M,C] = cast(x[M,C]) between fp32 and bf16; x / out may be channel slices (row-strided views)."""
    M, C, ldx = _rows(x)
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=dtype)
    check(lib().sniper_cast_rows(_ptr(x), ldx, _sdt(x), _ptr(out), _rows(out)[2], _sdt(out), M, C, _stream()))
    return out


class BNPool:
    """One device allocation for the state of every BatchNorm of a model (filled by ONE H2D copy instead of ~9 fill
    kernels per layer): per layer 6 float vectors [gamma? beta? moving_mean moving_var mean invstd scale shift] and a
    double[2C] statistics scratch."""

    def __init__(self, total_channels, device):
        self.device = device
        self.f = torch.zeros(8 * total_channels)         # host side until finalize()
        self.d_len = 4 * total_channels
        self.fo = 0
        self.do = 0
        self.pending = []

    def take(self, C, ones=False):
        o = self.fo
        self.fo += (C + 3) // 4 * 4          # keep every vector 16-byte aligned
        if ones:
            self.f[o:o + C] = 1.0
        return o

    def take_sums(self, C):
        o = self.do
        self.do += 2 * C
        return o

    def finalize(self):
        self.f = self.f[:max(self.fo, 1)].to(self.device)
        self.d = torch.zeros(max(self.do, 1), dtype=torch.float64, device=self.device)
        for fn in self.pending:
            fn()
        self.pending = []


class BNState:
    """Per-BN device state: parameters, moving statistics and the per-step (mean, invstd, scale, shift)."""

    def __init__(self, C, device, gamma=None, beta=None, dgamma=None, dbeta=None, pool=None):
        self.C = C
        self.dgamma, self.dbeta = dgamma, dbeta
        if pool is None:
            z = lambda: torch.zeros(C, device=device)
            self.gamma = gamma if gamma is not None else torch.ones(C, device=device)
            self.beta = beta if beta is not None else z()
            self.moving_mean, self.moving_var = z(), torch.ones(C, device=device)
            self.mean, self.invstd, self.scale, self.shift = z(), z(), z(), z()
            self.sums = torch.zeros(2 * C, dtype=torch.float64, device=device)
            self.sums_f = torch.zeros(2 * C, dtype=torch.float64, device=device)
            return
        og = pool.take(C, ones=True) if gamma is None else None
        ob = pool.take(C) if beta is None else None
        om, ov = pool.take(C), pool.take(C, ones=True)
        rest = [pool.take(C) for _ in range(4)]
        osum = pool.take_sums(C)
        osum_f = pool.take_sums(C)

        def bind():
            v = lambda o: pool.f[o:o + C]
            self.gamma = gamma if gamma is not None else v(og)
            self.beta = beta if beta is not None else v(ob)
            self.moving_mean, self.moving_var = v(om), v(ov)
            self.mean, self.invstd, self.scale, self.shift = [v(o) for o in rest]
            self.sums = pool.d[osum:osum + 2 * C]
            self.sums_f = pool.d[osum_f:osum_f + 2 * C]       # forward statistics accumulated by the producing conv
        pool.pending.append(bind)


def bn_stats(x, bn, eps=2e-5, momentum=0.9, fix_gamma=False, update_moving=True):
    """Train-mode BatchNorm statistics of x -> bn.(mean, invstd, scale, shift) (+ moving stats)."""
    M, C, ldx = _rows(x)
    check(lib().sniper_bn_stats(_ptr(x), ldx, M, C, _ptr(bn.gamma), _ptr(bn.beta), float(eps), float(momentum),
                                int(fix_gamma), _ptr(bn.moving_mean if update_moving else None),
                                _ptr(bn.moving_var if update_moving else None), _ptr(bn.sums), _ptr(bn.mean),
                                _ptr(bn.invstd), _ptr(bn.scale), _ptr(bn.shift), _sdt(x), _stream()))


def bn_finalize(bn, M, eps=2e-5, momentum=0.9, fix_gamma=False, update_moving=True):
    """Same as bn_stats when bn.sums was already accumulated by the producing conv's epilogue (stats=bn.sums)."""
    check(lib().sniper_bn_finalize(_ptr(bn.sums), M, bn.C, _ptr(bn.gamma), _ptr(bn.beta), float(eps), float(momentum),
                                   int(fix_gamma), _ptr(bn.moving_mean if update_moving else None),
                                   _ptr(bn.moving_var if update_moving else None), _ptr(bn.mean), _ptr(bn.invstd),
                                   _ptr(bn.scale), _ptr(bn.shift), _stream()))


def bn_apply_train(x, bn, eps=2e-5, momentum=0.9, relu=True, fix_gamma=False, update_moving=True, out=None):
    """relu?(bn_train(x)) when the statistics of x already sit in bn.sums_f (accumulated by the producing conv's
    epilogue): finalisation + apply in one launch.  bn.sums_f is left as is -- it is cleared by bn_param_grad_batched."""
    M, C, ldx = _rows(x)
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=x.dtype)
    check(lib().sniper_bn_apply_train(_ptr(x), ldx, _ptr(bn.sums_f), M, C, _ptr(bn.gamma), _ptr(bn.beta), float(eps),
                                      float(momentum), int(fix_gamma), _ptr(bn.moving_mean if update_moving else None),
                                      _ptr(bn.moving_var if update_moving else None), _ptr(bn.mean), _ptr(bn.invstd),
                                      _ptr(bn.scale), _ptr(bn.shift), _ptr(out), _rows(out)[2], int(relu), _sdt(x),
                                      _stream()))
    return out


def bn_frozen(bn, eps=2e-5, fix_gamma=False):
    check(lib().sniper_bn_frozen(bn.C, _ptr(bn.gamma), _ptr(bn.beta), _ptr(bn.moving_mean), _ptr(bn.moving_var),
                                 float(eps), int(fix_gamma), _ptr(bn.scale), _ptr(bn.shift), _stream()))


def bn_relu_bwd(x, dy, bn, add=None, out=None, defer=False):
    """Backward of relu(bn_train(x)); accumulates bn.dgamma / bn.dbeta; returns dx (+ add).
    defer=True leaves (s1, s2) in bn.sums for one bn_param_grad_batched call at the end of the backward pass."""
    M, C, ldx = _rows(x)
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=x.dtype)
    assert dy.dtype == x.dtype and out.dtype == x.dtype and (add is None or add.dtype == x.dtype)
    check(lib().sniper_bn_relu_bwd(_ptr(x), ldx, _ptr(dy), _rows(dy)[2], _ptr(bn.scale), _ptr(bn.shift), _ptr(bn.mean),
                                   _ptr(bn.invstd), _ptr(bn.sums), _ptr(add), 0 if add is None else _rows(add)[2],
                                   _ptr(out), _rows(out)[2], None if defer else _ptr(bn.dgamma),
                                   None if defer else _ptr(bn.dbeta), M, C, _sdt(x), _stream()))
    return out


def bn_act_bwd(x, dy, bn, act, add=None, out=None, defer=False):
    """Backward of act(bn_train(x)), act 1 = ReLU, 2 = clip(y, 0, 6), 3 = none; otherwise as bn_relu_bwd."""
    M, C, ldx = _rows(x)
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=x.dtype)
    assert dy.dtype == x.dtype and out.dtype == x.dtype and (add is None or add.dtype == x.dtype)
    check(lib().sniper_bn_act_bwd(_ptr(x), ldx, _ptr(dy), _rows(dy)[2], _ptr(bn.scale), _ptr(bn.shift), _ptr(bn.mean),
                                  _ptr(bn.invstd), _ptr(bn.sums), _ptr(add), 0 if add is None else _rows(add)[2],
                                  _ptr(out), _rows(out)[2], None if defer else _ptr(bn.dgamma),
                                  None if defer else _ptr(bn.dbeta), M, C, int(act), _sdt(x), _stream()))
    return out


def affine_relu_bwd(x, dy, scale, shift, add=None, relu=True, out=None):
    M, C, ldx = _rows(x)
    if out is None:
        out = torch.empty(x.shape, device=x.device)
    check(lib().sniper_affine_relu_bwd(_ptr(x), ldx, _ptr(dy), _rows(dy)[2], _ptr(scale), _ptr(shift), _ptr(add),
                                       0 if add is None else _rows(add)[2], _ptr(out), _rows(out)[2], M, C, int(relu),
                                       _stream()))
    return out


def relu_bwd(y, dy, out=None):
    M, C, ldy = _rows(y)
    if out is None:
        out = torch.empty(y.shape, device=y.device, dtype=y.dtype)
    assert dy.dtype == y.dtype and out.dtype == y.dtype
    check(lib().sniper_relu_bwd(_ptr(y), ldy, _ptr(dy), _rows(dy)[2], _ptr(out), _rows(out)[2], M, C, _sdt(y), _stream()))
    return out


def maxpool3x3s2(x):
    NB, H, W, C = x.shape
    y = torch.empty(NB, (H - 1) // 2 + 1, (W - 1) // 2 + 1, C, device=x.device, dtype=x.dtype)
    check(lib().sniper_maxpool3x3s2_nhwc(_ptr(x), _ptr(y), NB, H, W, C, _sdt(x), _stream()))
    return y


def stem_conv(x_nchw, w, in_scale, in_shift, out_scale, out_shift, out_dtype=torch.float32):
    """bn_data -> conv0 7x7/2 pad 3 -> bn0 -> relu; NCHW fp32 in, NHWC out (fp32 or bf16).  w: [64,7,7,3]."""
    NB, C, H, W = x_nchw.shape
    assert C == 3 and w.shape == (64, 7, 7, 3)
    y = torch.empty(NB, (H - 1) // 2 + 1, (W - 1) // 2 + 1, 64, device=x_nchw.device, dtype=out_dtype)
    check(lib().sniper_stem_conv(_ptr(x_nchw), _ptr(w), _ptr(in_scale), _ptr(in_shift), _ptr(out_scale),
                                 _ptr(out_shift), _ptr(y), NB, H, W, _sdt(y), _stream()))
    return y


def stem_rows(w, dtype=torch.float32):
    """conv0 weights [64,7,7,3] -> the B operand of the tensor-core stem: [64, Kp] rows in (kh, kw, c) order, zero-padded
    to the MMA's K granularity (160 fp32 / 192 bf16)."""
    Kp = 160 if dtype == torch.float32 else 192
    rows = torch.zeros(64, Kp, device=w.device, dtype=torch.float32)
    rows[:, :147] = w.reshape(64, 147)
    return rows.to(dtype)


def stem_conv_tc(x_nchw, rows, in_scale, in_shift, out_scale, out_shift, out_dtype=torch.float32):
    """The stem on the tensor cores: im2col of bn_data(x) (sniper_stem_im2col) + wgmma GEMM with bn0 + ReLU in the
    epilogue.  rows = stem_rows(conv0_w, dtype): fp32 rows run as TF32, bf16 rows as bf16 (fp32 accumulation)."""
    NB, C, H, W = x_nchw.shape
    assert C == 3 and rows.shape[0] == 64
    Ho, Wo, Kp = (H - 1) // 2 + 1, (W - 1) // 2 + 1, rows.shape[1]
    col = torch.empty(NB * Ho * Wo, Kp, device=x_nchw.device, dtype=rows.dtype)
    check(lib().sniper_stem_im2col(_ptr(x_nchw), _ptr(in_scale), _ptr(in_shift), _ptr(col), NB, H, W, Kp, _sdt(col),
                                   _stream()))
    y = gemm_nt(col, rows, scale=out_scale, bias=out_shift, relu=True, out_dtype=out_dtype)
    return y.view(NB, Ho, Wo, 64)


def weight_transpose(w, Cout, T, Cin, sel_dev, out=None):
    """w [Cout,T,Cin] -> [Cin, len(sel), Cout] with out[ci,j,co] = w[co, sel[j], ci] (data-gradient operand)."""
    Tsel = sel_dev.numel()
    if out is None:
        out = torch.empty(Cin, Tsel * Cout, device=w.device)
    check(lib().sniper_weight_transpose(_ptr(w), _ptr(out), Cout, T, Cin, Tsel, _ptr(sel_dev), _stream()))
    return out


def weight_transpose_jobs(jobs, device):
    """jobs: list of (w fp32, wt fp32|bf16, sel_dev, Cout, T, Cin).  Returns the device job table for
    weight_transpose_batched."""
    rows, b0 = [], 0
    for w, wt, sel, Cout, T, Cin in jobs:
        Tsel = sel.numel()
        assert w.dtype == torch.float32
        rows.append([w.data_ptr(), wt.data_ptr(), sel.data_ptr(), Cout, T, Cin, Tsel, b0, _sdt(wt)])
        b0 += ((Cin + 31) // 32) * ((Cout + 31) // 32) * Tsel
    return torch.tensor(rows, dtype=torch.int64, device=device), len(rows), b0


def weight_transpose_batched(table):
    t, n, blocks = table
    check(lib().sniper_weight_transpose_batched(_ptr(t), n, blocks, _stream()))


def bn_param_grad_jobs(states, device):
    """states: BNState objects whose backward ran with defer=True."""
    rows = [[b.sums.data_ptr(), 0 if b.dgamma is None else b.dgamma.data_ptr(),
             0 if b.dbeta is None else b.dbeta.data_ptr(), b.C, b.sums_f.data_ptr()] for b in states]
    return torch.tensor(rows, dtype=torch.int64, device=device), len(rows)


def bn_param_grad_batched(table):
    t, n = table
    check(lib().sniper_bn_param_grad_batched(_ptr(t), n, _stream()))


def colsum_accum(x, out):
    M, C, ldx = _rows(x)
    assert x.dtype == torch.float32 and out.dtype == torch.float32 and out.shape == (C,) and out.is_contiguous(), \
        "column sums read an fp32 [M, C] and add to an fp32 [C]"
    check(lib().sniper_colsum(_ptr(x), ldx, M, C, _ptr(out), _stream()))
    return out


def sgd_mom(w, mom, g, lr, wd, momentum, rescale=1.0):
    check(lib().sniper_sgd_mom(_ptr(w), _ptr(mom), _ptr(g), w.numel(), float(lr), float(wd), float(momentum),
                               float(rescale), _stream()))


def sgd_mom_dev(w, mom, g, hyper, lr_mult, wd_mult, momentum, rescale=1.0, w_bf16=None):
    """SGD-momentum with lr / wd read from the device buffer `hyper` = [lr, wd] (graph-replay safe schedule);
    w_bf16: optional bf16 shadow of the updated weights (multi_precision, optimizer_op-inl.h:377-404)."""
    check(lib().sniper_sgd_mom_dev(_ptr(w), _ptr(mom), _ptr(g), w.numel(), _ptr(hyper), float(lr_mult), float(wd_mult),
                                   float(momentum), float(rescale), _ptr(w_bf16), _stream()))


def count_valid(label, out, ignore=-1):
    check(lib().sniper_count_valid(_ptr(label), label.numel(), int(ignore), _ptr(out), _stream()))


def rpn_softmax_loss(score, label, A, grad_scale, valid_cnt, prob, dscore, loss_sum):
    """score/prob/dscore: NHWC [B,H,W,>=2A]; label [B, A*H*W] in (a,h,w) order."""
    B, H, W, _ = score.shape
    ld = score.stride(2)
    check(lib().sniper_rpn_softmax_loss(_ptr(score), ld, _ptr(label), B, H, W, A, float(grad_scale), _ptr(valid_cnt),
                                        _ptr(prob), prob.stride(2), _ptr(dscore), 0 if dscore is None else dscore.stride(2),
                                        _ptr(loss_sum), _stream()))


def rpn_smooth_l1_loss(pred, target, weight, C4, grad_scale, dpred, loss_sum):
    B, H, W, _ = pred.shape
    check(lib().sniper_rpn_smooth_l1_loss(_ptr(pred), pred.stride(2), _ptr(target), _ptr(weight), B, H, W, C4,
                                          float(grad_scale), _ptr(dpred), dpred.stride(2), _ptr(loss_sum), _stream()))


def softmax_ce(logits, label, K, grad_scale, valid_cnt, prob, grad, loss_sum, ignore=-1):
    N, ld = logits.shape[0], logits.stride(0)
    check(lib().sniper_softmax_ce(_ptr(logits), ld, _ptr(label), N, K, int(ignore), float(grad_scale), _ptr(valid_cnt),
                                  _ptr(prob), 0 if prob is None else prob.stride(0), _ptr(grad),
                                  0 if grad is None else grad.stride(0), _ptr(loss_sum), _stream()))


def smooth_l1_loss(pred, target, weight, C, grad_scale, grad, loss_sum):
    N, ld = pred.shape[0], pred.stride(0)
    check(lib().sniper_smooth_l1_loss(_ptr(pred), ld, _ptr(target), _ptr(weight), N, C, float(grad_scale), _ptr(grad),
                                      grad.stride(0), _ptr(loss_sum), _stream()))


def deform_im2col(x, offset, *, kh=3, kw=3, stride=1, dil=1, pad=1, dgroups=4, out=None):
    """Bilinear-sampled im2col (deformable_im2col.cuh:216-263): x [N,H,W,C], offset [N,Ho,Wo,>=dg*2*kh*kw]
    -> col [N*Ho*Wo, kh*kw*C] (tap-major)."""
    NB, H, W, C = x.shape
    Ho = (H + 2 * pad - dil * (kh - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (kw - 1) - 1) // stride + 1
    if out is None:
        out = torch.empty(NB * Ho * Wo, kh * kw * C, device=x.device, dtype=x.dtype)
    assert x.is_contiguous() and offset.dtype == torch.float32 and out.dtype == x.dtype
    check(lib().sniper_deform_im2col(_ptr(x), _ptr(offset), NB, H, W, C, kh, kw, stride, dil, pad, dgroups,
                                     offset.stride(2), _ptr(out), _sdt(x), _stream()))
    return out


def deform_col2im(dcol, x, offset, *, kh=3, kw=3, stride=1, dil=1, pad=1, dgroups=4, dx=None, doffset=None):
    """Transposes of deform_im2col: dx (accumulated, always fp32) and doffset (fp32)
    (deformable_im2col.cuh:317-360, 419-480).  dcol / x: fp32 or bf16."""
    NB, H, W, C = x.shape
    if dx is None:
        dx = torch.zeros(x.shape, device=x.device)
    if doffset is None:
        doffset = torch.zeros_like(offset)
    assert dcol.dtype == x.dtype and dx.dtype == torch.float32 and doffset.dtype == torch.float32
    acc = torch.zeros(x.shape, dtype=torch.float64, device=x.device)   # fp64 sums: reproducible dx
    check(lib().sniper_deform_col2im_fp64acc(_ptr(dcol), _ptr(x), _ptr(offset), NB, H, W, C, kh, kw, stride, dil, pad,
                                             dgroups, offset.stride(2), _ptr(dx), _ptr(doffset), _sdt(x), _ptr(acc),
                                             acc.numel(), _stream()))
    return dx, doffset


def anchor_target(gt_valid, ngt, gt_invalid, ninv, im_info, *, H=32, W=32, feat_stride=16,
                  scales=(2, 4, 7, 10, 13, 16, 24), ratios=(0.5, 1, 2), pos_thresh=0.5, neg_thresh=0.4, disable=None,
                  want_argmax=False):
    """RPN anchor matching of anchor_worker.worker (data_workers.py:194-363) for a whole chip batch.
    gt_valid [B,G,4] / gt_invalid [B,Gi,4] float32 (first ngt[b] / ninv[b] rows used, int32 counts),
    disable: optional uint8 [B,H*W*A] (the host's npr.choice subsampling).  Returns label [B,A*H*W],
    bbox_target, bbox_weight [B,4A,H,W] (+ argmax [B,H*W*A])."""
    B, G = gt_valid.shape[0], gt_valid.shape[1]
    Gi = gt_invalid.shape[1]
    A = len(scales) * len(ratios)
    dev = gt_valid.device
    label = torch.empty(B, A * H * W, device=dev)
    bt = torch.empty(B, 4 * A, H, W, device=dev)
    bw = torch.empty(B, 4 * A, H, W, device=dev)
    am = torch.empty(B, H * W * A, dtype=torch.int32, device=dev) if want_argmax else None
    scratch = torch.zeros(B * max(G, 1), dtype=torch.int64, device=dev)
    s, sp = _farr(scales)
    r, rp = _farr(ratios)
    check(lib().sniper_anchor_target(_ptr(gt_valid), _ptr(ngt), G, _ptr(gt_invalid), _ptr(ninv), Gi, _ptr(im_info),
                                     _ptr(disable), B, H, W, int(feat_stride), sp, len(s), rp, len(r), float(pos_thresh),
                                     float(neg_thresh), _ptr(scratch), _ptr(label), _ptr(bt), _ptr(bw), _ptr(am),
                                     _stream()))
    return (label, bt, bw, am) if want_argmax else (label, bt, bw)


def focus_label(boxes, nbox, *, H=32, W=32, feat_stride=16, dc_low=5.0, small_thresh=64.0, dc_high=90.0, out=None):
    """FocusPixel labels of gen_mask (data_workers.py:165-192) for a whole chip batch.  boxes [B,cap,4] float32: every
    GT box of the chip's image, shifted, scaled, rounded and clipped to the chip, first nbox[b] (int32) rows used.
    Returns scale_label [B, H*W] ((y,x) order, values 0 / 1 / -1)."""
    B, cap = boxes.shape[0], boxes.shape[1]
    assert boxes.dtype == torch.float32 and boxes.is_contiguous() and nbox.dtype == torch.int32
    if out is None:
        out = torch.empty(B, H * W, device=boxes.device)
    check(lib().sniper_focus_label(_ptr(boxes), _ptr(nbox), cap, B, H, W, int(feat_stride), float(dc_low),
                                   float(small_thresh), float(dc_high), _ptr(out), _stream()))
    return out


def focus_acc(prob, label, counts):
    """counts[0] += #(argmax(prob) == label), counts[1] += #(label != -1): prob [..., >=2] (the 2-channel softmax,
    channel stride prob.stride(-2)), label with one entry per row of prob."""
    n = label.numel()
    check(lib().sniper_focus_acc(_ptr(prob), prob.stride(-2), _ptr(label), n, _ptr(counts), _stream()))


def train_metric_workspace(device):
    """The zero-filled scratch sniper_train_metric_accum needs (reusable across launches and graph replays)."""
    return torch.zeros(int(lib().sniper_train_metric_workspace_bytes()), dtype=torch.uint8, device=device)


def train_metric_accum(rpn_prob, rpn_label, A, cls_prob, cls_label, counts, loss_buf, acc, workspace, af_prob=None,
                       af_label=None):
    """Adds one step's training-metric terms into `acc` (int64 [24]: num_inst[8] | hits[8] | float64 sum[8], see
    csrc/train_metric.cu).  rpn_prob NHWC [B,H,W,>=2A], rpn_label [B,A*H*W]; cls_prob [N,>=K] (K = its width),
    cls_label [N]; af_prob [B,Hf,Wf,>=2] / af_label [B,Hf*Wf] or None; counts int32 (count_valid results), loss_buf
    the step's loss sums."""
    B, H, W, _ = rpn_prob.shape
    N, K = cls_prob.shape
    assert acc.dtype == torch.int64 and acc.numel() == 24 and acc.is_contiguous() and counts.dtype == torch.int32
    Haf = Waf = ld_af = 0
    if af_prob is not None:
        Haf, Waf, ld_af = af_prob.shape[1], af_prob.shape[2], af_prob.stride(2)
    check(lib().sniper_train_metric_accum(_ptr(rpn_prob), rpn_prob.stride(2), _ptr(rpn_label), B, H, W, int(A),
                                          _ptr(cls_prob), cls_prob.stride(0), _ptr(cls_label), N, K,
                                          _ptr(af_prob), ld_af, _ptr(af_label), Haf, Waf,
                                          _ptr(counts), _ptr(loss_buf), _ptr(acc), _ptr(workspace), _stream()))


def soft_nms_batched(dets, offsets, *, sigma=0.55, Nt=0.3, threshold=0.001, method=2):
    """cpu_soft_nms (lib/nms/cpu_nms.pyx:17-110) on every segment dets[offsets[p]:offsets[p+1]] ([.,5] rows x1,y1,x2,y2,score)
    at once.  Returns (dets_out, counts): the first counts[p] rows of segment p are its surviving detections in the
    reference's output order, exact score ties included; `dets` itself is not modified."""
    assert dets.is_cuda and dets.dtype == torch.float32 and dets.dim() == 2 and dets.shape[1] == 5 and dets.is_contiguous()
    assert offsets.dtype == torch.int32 and offsets.is_cuda
    P = offsets.numel() - 1
    out = dets.clone()
    counts = torch.zeros(max(P, 1), dtype=torch.int32, device=dets.device)
    scratch = torch.empty((dets.shape[0], 6), dtype=torch.float32, device=dets.device)     # rows + compaction slots
    check(lib().sniper_soft_nms_batched(_ptr(out), _ptr(offsets), P, float(sigma), float(Nt), float(threshold), int(method),
                                        _ptr(counts), _ptr(scratch), _stream()))
    return out, counts[:P]


def proposal_nms_batched(dets, offsets):
    """nmsp (lib/nms/nms.py:48-80, IoU threshold 0.7) of every image p = rows dets[offsets[p]:offsets[p+1]] at once.
    dets: device float32 [total, 5] (x1, y1, x2, y2, score >= 0); offsets: host int32 [P+1], at most 4096 rows per
    image.  Returns (keep, counts) on the host: keep[offsets[p]:offsets[p] + counts[p]] are image p's kept rows (indices
    local to the image) in nmsp's keep order.  Waits for the launch."""
    assert dets.is_cuda and dets.dtype == torch.float32 and dets.dim() == 2 and dets.shape[1] == 5 and dets.is_contiguous()
    offsets = np.ascontiguousarray(offsets, dtype=np.int32)
    P = offsets.size - 1
    assert P >= 0 and offsets[-1] == dets.shape[0]
    off_dev = torch.from_numpy(offsets).to(dets.device)
    counts = torch.zeros(max(P, 1), dtype=torch.int32, device=dets.device)
    keep = torch.zeros(max(dets.shape[0], 1), dtype=torch.int32, device=dets.device)
    check(lib().sniper_proposal_nms_batched(_ptr(dets), _ptr(off_dev), offsets.ctypes.data, P, _ptr(counts), _ptr(keep),
                                            _stream()))
    counts = counts[:P].cpu().numpy()
    bad = np.where(counts < 0)[0]
    if len(bad):
        raise _libmod.SniperError("proposal_nms_batched: image %d has a negative score" % int(bad[0]))
    return keep.cpu().numpy(), counts


def detect_post_workspace(device):
    """The scratch `detect_post` needs (block counts of one launch); reusable by launches on the same stream."""
    return torch.empty(lib().sniper_detect_post_workspace_bytes() // 4, dtype=torch.int32, device=device)


def detect_post(rois, cls_prob, bbox_pred, im_info, chips, rows, keys, state, workspace, *, cls_thresh=1e-3, scale=0,
                rows_bound=0):
    """Tester.detect's box decoding, the score threshold / chip-border pruning of get_detections and the valid-range
    filter of aggregate (lib/inference.py:100-139, 232-351, 152-230) for one batch in one launch, no copy to the host.
    rois [B*R,5], cls_prob [B*R,K], bbox_pred [B*R,4] (any row stride: the view the R-FCN head returns), im_info
    [B,3]; chips: float64 [B,12] device table (`inference.chip_table`).  Surviving rows are appended to rows [cap,5] /
    keys [cap] (int64, `inference.pack_key`) at state[0] (int64 [2]: cursor, rows a refused launch needed).
    rows_bound: the caller's upper bound on the cursor; raises when rows_bound + B*R*(K-1) does not fit."""
    _f32(rois), _f32(cls_prob), _f32(im_info), _f32(rows)
    assert bbox_pred.is_cuda and bbox_pred.dtype == torch.float32 and bbox_pred.dim() == 2 and bbox_pred.shape[1] == 4 \
        and bbox_pred.stride(1) == 1, "bbox_pred: fp32 CUDA [N,4] with unit column stride"
    B, (N, K) = im_info.shape[0], cls_prob.shape
    assert B > 0 and N % B == 0 and rois.shape == (N, 5) and bbox_pred.shape[0] == N
    assert chips.is_cuda and chips.dtype == torch.float64 and chips.shape == (B, 12) and chips.is_contiguous()
    assert keys.is_cuda and keys.dtype == torch.int64 and keys.is_contiguous() and keys.numel() == rows.shape[0]
    assert rows.dim() == 2 and rows.shape[1] == 5 and state.is_cuda and state.dtype == torch.int64 and state.numel() == 2
    assert workspace.is_cuda and workspace.dtype == torch.int32
    check(lib().sniper_detect_post(_ptr(rois), _ptr(cls_prob), _ptr(bbox_pred), bbox_pred.stride(0), _ptr(im_info),
                                   _ptr(chips), B, N // B, K, float(cls_thresh), int(scale), _ptr(rows), _ptr(keys),
                                   rows.shape[0], int(rows_bound), _ptr(state), _ptr(workspace), _stream()))


# ---------------------------------------------------------------------------------------------
# COCO box evaluation (lib/dataset/pycocotools/cocoeval.py): a CSR over the non-empty (category, image) pairs; pair p
# owns GT rows gt_off[p]:gt_off[p+1] and score-sorted detection rows dt_off[p]:dt_off[p+1] (host int32 offsets)
# ---------------------------------------------------------------------------------------------
def _f64(t):
    assert t.is_cuda and t.dtype == torch.float64 and t.is_contiguous(), "expected contiguous float64 CUDA tensor"
    return t


def _off(off):
    off = np.ascontiguousarray(off, dtype=np.int32)
    assert off.ndim == 1 and off.size >= 1
    return off


def coco_box_iou_batched(dt_box, gt_box, gt_flags, dt_off, gt_off):
    """bbIou (maskApi.c:98-109) of every pair: returns (ious, iou_off) with pair p's [D_p, G_p] matrix (row d = the
    d-th detection) at ious[iou_off[p]:iou_off[p+1]] (device float64, host int64 offsets)."""
    dt_off, gt_off = _off(dt_off), _off(gt_off)
    P = dt_off.size - 1
    dev = dt_box.device
    iou_off = np.concatenate([[0], np.cumsum(np.diff(dt_off).astype(np.int64) * np.diff(gt_off))]).astype(np.int64)
    out = torch.empty(max(int(iou_off[-1]), 1), dtype=torch.float64, device=dev)
    d_dt, d_gt, d_iou = (torch.from_numpy(o).to(dev) for o in (dt_off, gt_off, iou_off))
    check(lib().sniper_coco_box_iou_batched(_ptr(_f64(dt_box)), _ptr(_f64(gt_box)), _ptr(gt_flags), _ptr(d_dt),
                                            _ptr(d_gt), _ptr(d_iou), dt_off.ctypes.data, gt_off.ctypes.data,
                                            iou_off.ctypes.data, P, _ptr(out), _stream()))
    return out, iou_off


def coco_match(dt_box, dt_area, dt_id, gt_box, gt_area, gt_flags, gt_id, dt_off, gt_off, iou_thrs, area_rng,
               full=False):
    """evaluateImg (cocoeval.py:189-272) of every pair x area range x IoU threshold in one launch.  gt_flags uint8:
    bit 0 iscrowd, bit 1 the annotation's `ignore`; ids int64.  Returns a dict of device tensors: dt_flags [A, T, Dtot]
    uint8 (bit 0 matched, bit 1 ignored), npig [P, A] int32, gt_match [A, T, Gtot] int64 (matching dt id in the
    ignore-sorted GT order), and with full=True also dt_match [A, T, Dtot] (matched gt id) and gt_order [A, Gtot]
    (pair-local GT index at each ignore-sorted position)."""
    dt_off, gt_off = _off(dt_off), _off(gt_off)
    P = dt_off.size - 1
    thr = np.ascontiguousarray(iou_thrs, dtype=np.float64)
    rng = np.ascontiguousarray(area_rng, dtype=np.float64).reshape(-1)
    T, A = thr.size, rng.size // 2
    Dtot, Gtot = int(dt_off[-1]), int(gt_off[-1])
    dev = dt_box.device
    assert gt_flags.dtype == torch.uint8 and dt_id.dtype == torch.int64 and gt_id.dtype == torch.int64
    r = dict(dt_flags=torch.empty(A, T, Dtot, dtype=torch.uint8, device=dev),
             npig=torch.empty(max(P, 1), A, dtype=torch.int32, device=dev),
             gt_match=torch.empty(A, T, Gtot, dtype=torch.int64, device=dev))
    if full:
        r.update(dt_match=torch.empty(A, T, Dtot, dtype=torch.int64, device=dev),
                 gt_order=torch.empty(A, Gtot, dtype=torch.int32, device=dev))
    d_dt, d_gt = torch.from_numpy(dt_off).to(dev), torch.from_numpy(gt_off).to(dev)
    check(lib().sniper_coco_match(_ptr(_f64(dt_box)), _ptr(_f64(dt_area)), _ptr(dt_id), _ptr(_f64(gt_box)),
                                  _ptr(_f64(gt_area)), _ptr(gt_flags), _ptr(gt_id), _ptr(d_dt), _ptr(d_gt),
                                  dt_off.ctypes.data, gt_off.ctypes.data, P, thr.ctypes.data, T, rng.ctypes.data, A,
                                  _ptr(r["dt_flags"]), _ptr(r["npig"]), _ptr(r["gt_match"]), _ptr(r.get("dt_match")),
                                  _ptr(r.get("gt_order")), _stream()))
    return r


def coco_category_order(dt_score, dt_cat):
    """The stable order of the detections by (category, descending score): cocoeval's
    np.argsort(-dtScores, kind='mergesort') over each category's concatenation (cocoeval.py:321-325), for all categories
    at once.  -0.0 counts as +0.0; NaN scores are refused."""
    s = _f64(dt_score) + 0.0
    if bool(torch.isnan(s).any()):
        raise ValueError("coco_category_order: a detection score is NaN")
    o1 = torch.sort(s, descending=True, stable=True).indices
    o2 = torch.sort(dt_cat[o1], stable=True).indices
    return o1[o2].to(torch.int32).contiguous()


def coco_accumulate(dt_flags, dt_rank, cat_order, dt_off, npig, cat_pair_off, max_dets, rec_thrs):
    """accumulate (cocoeval.py:274-374): precision [T, R, K, A, M] and recall [T, K, A, M] float64 (device), from
    coco_match's dt_flags / npig, each detection's rank in its pair (dt_rank int32), coco_category_order's cat_order,
    and cat_pair_off (host int32 [K+1]: the pairs of category k are cat_pair_off[k]:cat_pair_off[k+1])."""
    dt_off, cat_pair_off = _off(dt_off), _off(cat_pair_off)
    K, P = cat_pair_off.size - 1, dt_off.size - 1
    A, T = dt_flags.shape[0], dt_flags.shape[1]
    md = np.ascontiguousarray(max_dets, dtype=np.int32)
    rt = np.ascontiguousarray(rec_thrs, dtype=np.float64)
    M, R = md.size, rt.size
    dev = dt_flags.device
    precision = torch.empty(T, R, K, A, M, dtype=torch.float64, device=dev)
    recall = torch.empty(T, K, A, M, dtype=torch.float64, device=dev)
    d_dt, d_cat = torch.from_numpy(dt_off).to(dev), torch.from_numpy(cat_pair_off).to(dev)
    check(lib().sniper_coco_accumulate(_ptr(dt_flags), _ptr(dt_rank), _ptr(cat_order), _ptr(d_dt), _ptr(npig),
                                       _ptr(d_cat), dt_off.ctypes.data, cat_pair_off.ctypes.data, K, P, A, T,
                                       md.ctypes.data, M, rt.ctypes.data, R, _ptr(precision), _ptr(recall),
                                       _stream()))
    return precision, recall


# ---------------------------------------------------------------------------------------------
# MobileNetV2 layers (symbols/faster/mobilenetv2_e2e.py): depthwise 3x3, first-layer im2col, shortcut add
# ---------------------------------------------------------------------------------------------
def depthwise3x3(x, w, stride=1, out=None):
    """x: [N,H,W,C] (fp32 | bf16), w: [9,C] fp32 tap-major -> [N,Ho,Wo,C]; pad 1.  x and out may be channel slices."""
    NB, H, W, C = x.shape
    assert w.shape == (9, C) and w.dtype == torch.float32 and w.is_contiguous()
    ldx = _pixel_ld(x)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    if out is None:
        out = torch.empty(NB, Ho, Wo, C, device=x.device, dtype=x.dtype)
    assert out.dtype == x.dtype and out.shape == (NB, Ho, Wo, C)
    check(lib().sniper_depthwise3x3_fwd(_ptr(x), ldx, _ptr(w), _ptr(out), _pixel_ld(out), NB, H, W, C, stride, _sdt(x),
                                        _stream()))
    return out


def depthwise3x3_dgrad(dy, w, in_hw, stride=1, out=None):
    """dx [N,H,W,C] of depthwise3x3 for dy [N,Ho,Wo,C].  dy and out may be channel slices."""
    NB, Ho, Wo, C = dy.shape
    H, W = in_hw
    assert (H - 1) // stride + 1 == Ho and (W - 1) // stride + 1 == Wo
    assert w.shape == (9, C) and w.dtype == torch.float32 and w.is_contiguous()
    lddy = _pixel_ld(dy)
    if out is None:
        out = torch.empty(NB, H, W, C, device=dy.device, dtype=dy.dtype)
    assert out.dtype == dy.dtype and out.shape == (NB, H, W, C)
    check(lib().sniper_depthwise3x3_dgrad(_ptr(dy), lddy, _ptr(w), _ptr(out), _pixel_ld(out), NB, H, W, C, stride,
                                          _sdt(dy), _stream()))
    return out


def depthwise3x3_wgrad(x, dy, dw, stride=1):
    """dw[9,C] (fp32) += correlation of dy with the shifted input, summed in a fixed order (two calls give the same
    bits)."""
    NB, H, W, C = x.shape
    assert dw.shape == (9, C) and dw.dtype == torch.float32 and dw.is_contiguous() and x.dtype == dy.dtype
    assert x.is_contiguous() and dy.is_contiguous()
    _stream_workspace()
    check(lib().sniper_depthwise3x3_wgrad(_ptr(x), x.stride(2), _ptr(dy), dy.stride(2), _ptr(dw), NB, H, W, C, stride,
                                          _sdt(x), _stream()))
    return dw


def im2col3x3s2(x_nchw, Kp, dtype=torch.float32, out=None):
    """[N,3,H,W] fp32 -> [N,Ho,Wo,Kp] rows of the first layer's 3x3 / stride-2 patches, K order (kh, kw, ci)."""
    NB, Cin, H, W = x_nchw.shape
    assert x_nchw.dtype == torch.float32 and x_nchw.is_contiguous()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    if out is None:
        out = torch.empty(NB, Ho, Wo, Kp, device=x_nchw.device, dtype=dtype)
    assert out.shape == (NB, Ho, Wo, Kp) and out.is_contiguous()
    check(lib().sniper_im2col3x3s2_nchw(_ptr(x_nchw), _ptr(out), NB, H, W, Cin, Kp, _sdt(out), _stream()))
    return out


def add_rows(a, b, out=None):
    M, C, lda = _rows(a)
    if out is None:
        out = torch.empty(a.shape, device=a.device, dtype=a.dtype)
    assert a.dtype == b.dtype == out.dtype and a.shape == b.shape
    check(lib().sniper_add_rows(_ptr(a), lda, _ptr(b), _rows(b)[2], _ptr(out), _rows(out)[2], M, C, _sdt(a), _stream()))
    return out


# ---------------------------------------------------------------------------------------------
# PASCAL VOC box evaluation (lib/dataset/pascal_voc_eval.py:73-181): detections class-major in the host's
# np.argsort(-confidence) order, GTs a CSR over the (class, image) pairs p = c * num_images + i (host int32 offsets)
# ---------------------------------------------------------------------------------------------
def voc_match(det_box, det_pair, gt_box, gt_difficult, gt_off, thresholds):
    """The matching loop of voc_eval (pascal_voc_eval.py:137-171) for every (class, image) pair and every overlap
    threshold in one launch.  det_box: [N, 4] float64 device, the results file's boxes in sorted order; det_pair: host
    int array [N], the pair of each sorted position; gt_box [G, 4] float64 and gt_difficult [G] uint8 device, in the
    CSR order of gt_off (host [P+1]).  Returns flags [T, N] uint8 (1 tp, 2 fp, 0 a hit on a difficult GT)."""
    gt_off = _off(gt_off)
    P = gt_off.size - 1
    thr = np.ascontiguousarray(thresholds, dtype=np.float64).reshape(-1)
    T = thr.size
    det_pair = np.ascontiguousarray(det_pair, dtype=np.int64).reshape(-1)
    N, G = det_pair.size, int(gt_off[-1])
    if N and (det_pair.min() < 0 or det_pair.max() >= P):
        raise ValueError("voc_match: a detection's pair index is outside [0, %d)" % P)
    if tuple(det_box.shape) != (N, 4) or tuple(gt_box.shape) != (G, 4) or tuple(gt_difficult.shape) != (G,):
        raise ValueError("voc_match: det_box must be [N, 4], gt_box [G, 4] and gt_difficult [G] (N = %d, G = %d)"
                         % (N, G))
    assert gt_difficult.dtype == torch.uint8
    # every pair's sorted positions in increasing order
    pos = np.argsort(det_pair, kind="stable").astype(np.int32)
    pair_off = np.zeros(P + 1, np.int32)
    np.cumsum(np.bincount(det_pair, minlength=P), out=pair_off[1:])
    dev = gt_box.device
    flags = torch.empty(T, N, dtype=torch.uint8, device=dev)
    taken = torch.empty(T, max(G, 1), dtype=torch.uint8, device=dev)
    d_pair, d_pos, d_gt = (torch.from_numpy(a).to(dev) for a in (pair_off, pos, gt_off))
    check(lib().sniper_voc_match(_ptr(_f64(det_box)), _ptr(d_pair), _ptr(d_pos), _ptr(_f64(gt_box)),
                                 _ptr(gt_difficult.contiguous()), _ptr(d_gt), pair_off.ctypes.data, gt_off.ctypes.data,
                                 P, thr.ctypes.data, T, _ptr(flags), _ptr(taken), _stream()))
    return flags


def voc_accumulate(flags, det_off, npos, use_07_metric, thresholds_07=None):
    """pascal_voc_eval.py:173-179 and voc_ap (:39-70) for every class and threshold, one block each: rec and prec
    [T, N] float64 (class c at det_off[c]:det_off[c+1], host [C+1]) and ap [T, C] float64, all on the device.  npos:
    [C] int32 device, the non-difficult GT count of each class.  The 11-point metric takes its recall thresholds from
    the host (default np.arange(0., 1.1, 0.1)); the area metric sums in numpy's pairwise order."""
    det_off = _off(det_off)
    C = det_off.size - 1
    T, N = flags.shape
    if int(det_off[-1]) != N:
        raise ValueError("voc_accumulate: det_off ends at %d, flags hold %d positions" % (det_off[-1], N))
    t07 = np.ascontiguousarray(np.arange(0., 1.1, 0.1) if thresholds_07 is None else thresholds_07, dtype=np.float64)
    dev = flags.device
    assert npos.dtype == torch.int32 and tuple(npos.shape) == (C,)
    rec = torch.empty(T, N, dtype=torch.float64, device=dev)
    prec = torch.empty(T, N, dtype=torch.float64, device=dev)
    ap = torch.empty(T, C, dtype=torch.float64, device=dev)
    terms = None if use_07_metric else torch.empty(T, N + C, dtype=torch.float64, device=dev)
    d_off = torch.from_numpy(det_off).to(dev)
    check(lib().sniper_voc_accumulate(_ptr(flags.contiguous()), _ptr(d_off), _ptr(npos.contiguous()),
                                      det_off.ctypes.data, C, T, int(bool(use_07_metric)), t07.ctypes.data, t07.size,
                                      _ptr(rec), _ptr(prec), _ptr(ap), _ptr(terms), _stream()))
    return rec, prec, ap


RECALL_RANGES = 7
_RECALL_DTYPES = {np.dtype(np.uint16): 0, np.dtype(np.float32): 1, np.dtype(np.float64): 2}


def proposal_recall(prop_box, prop_off, gt_box, gt_off, gt_range, thresholds, device="cuda",
                    max_workspace_bytes=1 << 30):
    """The matching and the statistics of IMDB.evaluate_recall (lib/dataset/imdb.py:291-397) on the device.

    prop_box: host [N, 4] uint16, float32 or float64, every image's proposals as stored (image i at
    prop_off[i]:prop_off[i+1]); gt_box: host [G, 4], the GTs the reference keeps, widened to float64 (image i at
    gt_off[i]:gt_off[i+1]); gt_range: host [G] uint8, bit r set when the GT's area (in its own dtype) lies in area range
    r (0 = all, 1 .. 6 = 0-25 .. 300-inf); thresholds: host float64 [T].  Pairs whose IoU matrix does not fit in shared
    memory use a device workspace, run in launches of at most `max_workspace_bytes` each (a single larger pair still
    runs).  Returns a dict of host arrays at full precision: recalls [7, T], ar [7], num_pos [7], gt_overlaps (7 sorted
    float64 arrays), area_counts [6] (proposals per range 1 .. 6), area_fraction [6] and avg_proposals."""
    prop_off, gt_off = _off(prop_off), _off(gt_off)
    I = prop_off.size - 1
    if gt_off.size != I + 1:
        raise ValueError("proposal_recall: prop_off and gt_off must have one entry per image plus one (%d, %d)"
                         % (prop_off.size, gt_off.size))
    prop_box, gt_box = np.asarray(prop_box), np.asarray(gt_box)
    if prop_box.dtype not in _RECALL_DTYPES:
        raise ValueError("proposal_recall: proposals must be uint16, float32 or float64, not %s" % prop_box.dtype)
    N, G = int(prop_off[-1]), int(gt_off[-1])
    if prop_box.shape != (N, 4) or gt_box.shape != (G, 4):
        raise ValueError("proposal_recall: prop_box must be [N, 4] and gt_box [G, 4] (N = %d, G = %d), not %s and %s"
                         % (N, G, prop_box.shape, gt_box.shape))
    if gt_box.dtype != np.float64:
        raise ValueError("proposal_recall: gt_box must be float64, not %s" % gt_box.dtype)
    if not (np.isfinite(prop_box).all() and np.isfinite(gt_box).all()):
        raise ValueError("proposal_recall: box coordinates must be finite")
    gt_range = np.ascontiguousarray(gt_range, dtype=np.uint8).reshape(-1)
    if gt_range.size != G:
        raise ValueError("proposal_recall: gt_range must hold one mask per GT (%d), not %d" % (G, gt_range.size))
    thr = np.asarray(thresholds)
    if thr.ndim != 1 or thr.dtype != np.float64:
        raise ValueError("proposal_recall: thresholds must be a 1-D float64 array")
    thr = np.ascontiguousarray(thr)
    T = thr.size
    prop_box, gt_box = np.ascontiguousarray(prop_box), np.ascontiguousarray(gt_box)
    L = lib()
    P = RECALL_RANGES * I
    ws_off = np.zeros(P + 1, np.int64)
    check(L.sniper_proposal_recall_workspace_bytes(prop_off.ctypes.data, gt_off.ctypes.data, gt_range.ctypes.data, I,
                                                   ws_off.ctypes.data))
    # per (range, image): the GTs in range, and what the image adds to gt_overlaps (nothing without proposals)
    bits = ((gt_range[:, None] >> np.arange(RECALL_RANGES, dtype=np.uint8)) & 1).astype(np.int64)
    cs = np.vstack([np.zeros((1, RECALL_RANGES), np.int64), np.cumsum(bits, axis=0)])
    m = (cs[gt_off[1:]] - cs[gt_off[:-1]]).T                              # [7, I]
    contrib = np.where(np.diff(prop_off)[None, :] > 0, m, 0)
    out_off = np.zeros(P + 1, np.int64)
    np.cumsum(contrib.reshape(-1), out=out_off[1:])
    num_pos = m.sum(axis=1).astype(np.int64)
    range_off = np.ascontiguousarray(out_off[::I] if I else np.zeros(RECALL_RANGES + 1, np.int64))

    dev = torch.device(device)
    up = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    d_prop = up(prop_box.view(np.int16) if prop_box.dtype == np.uint16 else prop_box)
    d_gt, d_range = up(gt_box), up(gt_range)
    d_poff, d_goff, d_out_off, d_ws_off = up(prop_off), up(gt_off), up(out_off), up(ws_off)
    overlaps = torch.empty(max(int(out_off[-1]), 1), dtype=torch.float64, device=dev)
    status = torch.zeros(max(P, 1), dtype=torch.uint8, device=dev)
    chunks, b = [], 0
    while b < P:
        e = int(np.searchsorted(ws_off, ws_off[b] + max_workspace_bytes, side="right")) - 1
        e = min(max(e, b + 1), P)
        chunks.append((b, e))
        b = e
    ws_need = max([int(ws_off[e] - ws_off[b]) for b, e in chunks] + [0])
    ws = torch.empty(ws_need, dtype=torch.uint8, device=dev) if ws_need else None
    dt = _RECALL_DTYPES[prop_box.dtype]
    with torch.cuda.device(dev):
        st = _stream()
        for b, e in chunks:
            check(L.sniper_proposal_recall_match(_ptr(d_prop), dt, _ptr(d_poff), _ptr(d_gt), _ptr(d_range),
                                                 _ptr(d_goff), _ptr(d_out_off), _ptr(d_ws_off), prop_off.ctypes.data,
                                                 gt_off.ctypes.data, gt_range.ctypes.data, ws_off.ctypes.data, I, b, e,
                                                 _ptr(ws), _ptr(overlaps), _ptr(status), st))
        counts = torch.empty(RECALL_RANGES * T + 6, dtype=torch.int64, device=dev)
        done = torch.empty(1, dtype=torch.int32, device=dev)
        recalls = torch.empty(max(RECALL_RANGES * T, 1), dtype=torch.float64, device=dev)
        ar = torch.empty(RECALL_RANGES, dtype=torch.float64, device=dev)
        hist = torch.empty(7, dtype=torch.float64, device=dev)
        d_thr = up(thr) if T else None
        check(L.sniper_proposal_recall_accumulate(_ptr(overlaps), range_off.ctypes.data, num_pos.ctypes.data,
                                                  _ptr(d_thr), T, _ptr(d_prop), dt, N, I, _ptr(counts), _ptr(done),
                                                  _ptr(recalls), _ptr(ar), _ptr(hist), st))
    bad = np.flatnonzero(status.cpu().numpy()[:P])
    if bad.size:
        p = int(bad[0])
        why = {1: "its best overlap is negative", 2: "an IoU has a zero union"}[int(status[p])]
        raise ValueError("proposal_recall: image %d, area range %d: %s (the reference asserts / divides by zero)"
                         % (p % I, p // I, why))
    ov = overlaps.cpu().numpy()
    cnt = counts.cpu().numpy()
    h = hist.cpu().numpy()
    return dict(recalls=recalls.cpu().numpy()[:RECALL_RANGES * T].reshape(RECALL_RANGES, T), ar=ar.cpu().numpy(),
                num_pos=num_pos, gt_overlaps=[np.sort(ov[range_off[r]:range_off[r + 1]])
                                              for r in range(RECALL_RANGES)],
                area_counts=cnt[RECALL_RANGES * T:].astype(np.int64), area_fraction=h[:6],
                avg_proposals=float(h[6]))


# ---------------------------------------------------------------------------------------------
# AutoFocus FocusChips (lib/chips/chips_inference.py:12-173)
# ---------------------------------------------------------------------------------------------
FOCUS_TABLE_COLS = 12


def focus_threshold(thresh):
    """The float32 t for which `v >= t` in float32 equals numpy's `float32 map >= thresh` for every float32 v: a Python
    float or int compares in float32 (t = float32(thresh)); a numpy float64 compares in double, which for float32 values
    is the comparison with the least float32 not below thresh."""
    t = np.float32(thresh)
    if np.result_type(np.float32, thresh) != np.float32 and float(t) < float(thresh):
        t = np.nextafter(t, np.float32(np.inf))
    return t


def focus_chips_table(maps, index, geometry):
    """The int64 [n, 12] table of `sniper_focus_chips` (validated): see `focus_chips` for maps / index / geometry."""
    index = np.asarray(index)
    geometry = np.asarray(geometry)
    if index.ndim != 2 or index.shape[1] != 6 or index.dtype.kind not in "iu":
        raise ValueError("focus_chips: index must be an integer [n, 6] array, not %s %s" % (index.dtype, index.shape))
    n = index.shape[0]
    if geometry.shape != (n, 5) or geometry.dtype != np.float64:
        raise ValueError("focus_chips: geometry must be float64 [%d, 5], not %s %s" % (n, geometry.dtype, geometry.shape))
    if not (np.isfinite(geometry).all() and (geometry[:, 2] > 0).all()):
        raise ValueError("focus_chips: geometry must be finite with a positive cscale")
    if not maps:
        if n:
            raise ValueError("focus_chips: %d maps refer to no tensor" % n)
        return np.zeros((0, FOCUS_TABLE_COLS), np.int64)
    dev = maps[0].device
    for k, t in enumerate(maps):
        if not (torch.is_tensor(t) and t.is_cuda and t.device == dev and t.dtype == torch.float32 and t.dim() == 3):
            raise ValueError("focus_chips: maps[%d] must be a float32 [B, H, W] tensor on %s" % (k, dev))
    index = index.astype(np.int64)
    ti, row, H, W, iw, ih = index.T
    if n and (ti.min() < 0 or ti.max() >= len(maps)):
        raise ValueError("focus_chips: index names a tensor outside maps[0:%d]" % len(maps))
    shape = np.array([t.shape for t in maps], np.int64).reshape(-1, 3)
    stride = np.array([t.stride() for t in maps], np.int64).reshape(-1, 3)
    base = np.array([t.data_ptr() for t in maps], np.int64)
    if n and ((row < 0) | (row >= shape[ti, 0]) | (H < 0) | (H > shape[ti, 1]) | (W < 0) | (W > shape[ti, 2])).any():
        raise ValueError("focus_chips: a map's row / H / W lies outside its tensor")
    if n and ((iw < 0) | (ih < 0)).any():
        raise ValueError("focus_chips: iw / ih must not be negative")
    if n and ((base[ti] == 0) & (H * W > 0)).any():
        raise ValueError("focus_chips: a map's tensor has a null address")
    table = np.zeros((n, FOCUS_TABLE_COLS), np.int64)
    table[:, 0] = base[ti] + row * stride[ti, 0] * 4
    table[:, 1], table[:, 2] = stride[ti, 1], stride[ti, 2]
    table[:, 3:7] = index[:, 2:6]
    table[:, 7:12] = np.ascontiguousarray(geometry).view(np.int64)
    return table


def focus_chips(maps, index, geometry, *, d, thresh, ms, capacity=8):
    """gmask (lib/chips/chips_inference.py:12-89) and the crop shift of add_chips (:158-162) for many FocusPixel maps in
    one `sniper_focus_chips` launch, the maps read in place.

    maps: device float32 tensors [B, Hc, Wc] (any strides: the `focus_map` view is fine); index: host int64 [n, 6] per map
    (tensor, row, H, W, iw, ih): map m is maps[tensor][row, :H, :W] and iw / ih are gmask's ceil(im_width / 16) /
    ceil(im_height / 16); geometry: host float64 [n, 5] per map (im_width, im_height, cscale, crop x1, crop y1).
    d, thresh, ms: the scale's CHIP_HYPERPARAMS.  Returns (chips, offsets): host float64 [total, 4] and int64 [n + 1], map
    m's FocusChips in image coordinates and gmask's order at chips[offsets[m]:offsets[m + 1]].  Waits for the launch; maps
    with more than `capacity` chips run once more with room for all of them."""
    if int(d) != d or d < 1 or int(ms) != ms or ms < 0:
        raise ValueError("focus_chips: d (%r) must be an integer >= 1 and ms (%r) an integer >= 0" % (d, ms))
    maps = list(maps)
    table = focus_chips_table(maps, index, geometry)
    n = table.shape[0]
    if n == 0:
        return np.zeros((0, 4)), np.zeros(1, np.int64)
    dev = maps[0].device
    H, W = table[:, 3], table[:, 4]
    L = lib()
    ws_off = np.zeros(n + 1, np.int64)
    check(L.sniper_focus_chips_workspace_bytes(table.ctypes.data, n, ws_off.ctypes.data))
    cap = max(int(capacity), 1)
    up = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    with torch.cuda.device(dev):
        d_table, d_ws_off = up(table), up(ws_off)
        ws = torch.empty(int(ws_off[-1]), dtype=torch.uint8, device=dev) if ws_off[-1] else None
        chips = torch.empty((max(n, 1), cap, 4), dtype=torch.float64, device=dev)
        counts = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        check(L.sniper_focus_chips(_ptr(d_table), _ptr(d_ws_off), table.ctypes.data, ws_off.ctypes.data, n, int(d),
                                   float(focus_threshold(thresh)), int(ms), _ptr(ws), cap, _ptr(chips), _ptr(counts),
                                   _stream()))
        cnt = counts.cpu().numpy()[:n].astype(np.int64)
        got = chips.cpu().numpy()
    bad = np.flatnonzero(cnt < 0)
    if bad.size:
        m = int(bad[0])
        why = {-1: "the merge loop did not settle within H * W + 2 passes",
               -2: "the table disagrees with its workspace offsets"}[int(cnt[m])]
        raise _libmod.SniperError("focus_chips: map %d (%d x %d): %s" % (m, H[m], W[m], why))
    off = np.zeros(n + 1, np.int64)
    np.cumsum(cnt, out=off[1:])
    out = np.empty((int(off[-1]), 4))
    over = cnt > cap
    m_i, k_i = np.nonzero((np.arange(cap)[None, :] < cnt[:, None]) & ~over[:, None])
    out[off[m_i] + k_i] = got[m_i, k_i]
    if over.any():
        sel = np.flatnonzero(over)
        more, more_off = focus_chips(maps, np.asarray(index)[sel], np.asarray(geometry)[sel], d=d, thresh=thresh, ms=ms,
                                     capacity=int(cnt[sel].max()))
        for q, m in enumerate(sel):
            out[off[m]:off[m + 1]] = more[more_off[q]:more_off[q + 1]]
    return out, off
