"""Regenerates include/sniper_b200.h from the extern "C" definitions in sniper_b200/csrc/*.cu|cpp plus the
reference citations below (kept here so that the header and the sources cannot drift apart)."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DOC = {
    "sniper_last_error": "Thread-local message of the last failing call.  Mirrors MXGetLastError (SNIPER-mxnet/include/mxnet/c_api.h:196-204).",
    "sniper_abi_version": "ABI version of this library (bumped on any signature change).",
    "sniper_stream_workspace_bytes": "Size of the fixed part of a stream workspace: the split-K parked partials and arrival counters of sniper_conv2d_wgrad_nhwc and the block-partial slab of sniper_depthwise3x3_wgrad, each 256-byte aligned, in this order; the tf32 operand copy area (sniper_conv2d_wgrad_scratch_bytes) follows it.",
    "sniper_set_stream_workspace": "Registers a caller-owned device buffer (256-byte aligned, at least sniper_stream_workspace_bytes() bytes, must outlive later launches) as the workspace of the launches on one (device, stream); registering again replaces it. Its counter region must be zero when it is registered; the kernels leave it zero. The library itself never allocates device memory.",
    "sniper_multi_proposal_target_workspace_bytes": "Scratch bytes for sniper_multi_proposal_target_fwd: replaces ResourceRequest::kTempSpace of MultiProposalTargetProp (multi_proposal_target-inl.h:143-146).",
    "sniper_generate_anchors": "Host helper, utils::GenerateAnchors (multi_proposal_target.cu:75-114): out[nr*ns,4], ratio-major.",
    "sniper_proposal_decode": "K1: utils::getProps (multi_proposal_target.cu:263-331). Anchor shift + bbox_transform_inv + clip + min-size / valid-range filters -> SoA boxes float4[B*A*H*W], score, area. layout 0 = NCHW (reference), 1 = NHWC (channel strides given).",
    "sniper_multi_proposal_target_fwd": "Drop-in for MultiProposalTargetGPUOp::Forward (multi_proposal_target.cu:362-589; operator surface multi_proposal_target-inl.h:55-177: arguments cls_prob,bbox_pred,im_info,gt_boxes,valid_ranges -> outputs rois,label,bbox_target,bbox_weight). Decode + greedy NMS (reference tie order) + GT append + IoU/label/target assignment, entirely on device: no D2H/H2D, no sync, no allocation. keep_idx/num_kept are optional parity outputs. Backward of the reference operator is a zero fill (cu:591-615) and needs no entry point.",
    "sniper_multi_proposal_workspace_bytes": "Scratch bytes for sniper_multi_proposal_fwd.",
    "sniper_multi_proposal_fwd": "Drop-in for the inference proposal operator MultiProposal (multi_proposal-inl.h:55-167: arguments cls_prob,bbox_pred,im_info -> outputs output(rois),score; CPU op multi_proposal.cc:273-374, GPU-build op multi_proposal.cu:400-631, which is host code with D2H copies). Decode + min-size filter + exact top-pre_nms_top_n selection + greedy NMS on device; flags 1 = the GPU build's anchor-type suppression. Rows after the kept ones: deterministic filler instead of the reference's rand() boxes.",
    "sniper_deform_psroi_fwd": "DeformablePSROIPoolingOp::Forward (contrib/deformable_psroi_pooling-inl.h:84-125, kernel .cu:71-161). top_count optional (hidden output of the reference), sample_idx optional parity output [count, spp^2, 4].",
    "sniper_deform_psroi_bwd": "DeformablePSROIPoolingOp::Backward (contrib/deformable_psroi_pooling-inl.h:127-174, kernel .cu:203-330). data_diff/trans_diff are accumulated into (kAddTo); zero them for kWriteTo.",
    "sniper_deform_psroi_bwd_fp64acc": "sniper_deform_psroi_bwd on the NHWC kernels with the gradients summed in a caller-owned fp64 scratch (reproducible run to run); -2 if the shape does not qualify.",
    "sniper_psroi_fwd": "PSROIPoolingOp::Forward (contrib/psroi_pooling.cu:51-118). bins optional parity output [count,4] = hstart,hend,wstart,wend.",
    "sniper_psroi_bwd": "PSROIPoolingOp::Backward (contrib/psroi_pooling.cu:146-210); accumulates into data_diff.",
    "sniper_gemm_nt": "C[M,N] = epi(A[M,K] * B[N,K]^T) on wgmma (register accumulators, TMA operands). Replaces FullyConnected -> cuBLAS (nn/fully_connected-inl.h) and linalg_gemm (contrib/deformable_convolution-inl.h:148-160). dtype 0 = fp32 storage / TF32 math, 1 = bf16. epi: *scale[n], +bias[n], +residual[m,n], relu; accumulate = red.global.add (fp32 outputs only; refused with out_bf16).",
    "sniper_gemm_plan": "Host-only: the tile width, ring depth, persistent grid and tail split sniper_gemm_nt would choose for a shape (no GPU needed).",
    "sniper_conv2d_nhwc": "NHWC implicit-GEMM convolution on wgmma; also the stride-1/stride-2 data gradient (flipped / parity-split weights, strided output map). Replaces cudnnConvolutionForward / BackwardData (nn/cudnn/cudnn_convolution-inl.h:144,211-266).",
    "sniper_conv2d_wgrad_nhwc": "Weight gradient dW[Cout, taps*Cin] += dY^T * im2col(X) on wgmma with split-K: bf16 reads the MN-major operands in place, tf32 first copies them channel-major into the copy area of the stream's workspace. Splits > 1 and the copies need the workspace (sniper_set_stream_workspace; refused without one, or with too small a copy area). Replaces cudnnConvolutionBackwardFilter (nn/cudnn/cudnn_convolution-inl.h:211-266).",
    "sniper_conv2d_wgrad_scratch_bytes": "Host-only: bytes of the tf32 operand copy area sniper_conv2d_wgrad_nhwc needs in the stream's workspace for a geometry (0 for bf16).",
    "sniper_affine_act": "y = act(x*scale[c] + shift[c]) on [M,C] rows (BatchNorm apply + Activation; nn/batch_norm.cu:658-700); relu 0 = none, 1 = ReLU, 2 = clip(y, 0, 6).",
    "sniper_bn_stats": "Train-mode BatchNorm statistics -> mean, invstd, scale, shift and moving statistics (cuDNN convention, nn/cudnn/cudnn_batch_norm-inl.h).",
    "sniper_bn_apply_train": "BatchNorm(train) + Activation in one launch when the input statistics were accumulated by the producing conv's epilogue: finalisation (mean / invstd / scale / shift / moving statistics, nn/batch_norm.cu:658-700 semantics) folded into the apply pass.",
    "sniper_bn_frozen": "use_global_stats BatchNorm: scale/shift from the moving statistics (nn/batch_norm.cu:671-674 path).",
    "sniper_bn_relu_bwd": "Backward of relu(bn_train(x)): dx (+add), dgamma +=, dbeta +=.",
    "sniper_bn_act_bwd": "Backward of act(bn_train(x)) with act 1 = ReLU (Activation), 2 = clip(y, 0, 6) (mx.sym.clip: relu6 of symbols/faster/mobilenetv2_e2e.py:18-19, gradient mask of tensor/matrix_op-inl.h:1319-1332), 3 = none (linear bottleneck): dx (+add), dgamma +=, dbeta +=.",
    "sniper_affine_relu_bwd": "Backward of relu?(x*scale+shift) for frozen BN.",
    "sniper_depthwise3x3_fwd": "Depthwise 3x3 convolution, pad 1, stride 1|2, NHWC, weights [9,C] fp32: Convolution(num_group = num_filter = C) of mobilenetv2_e2e.py:58-66 (src/operator/nn/depthwise_convolution-inl.h DepthwiseConvolutionOp::Forward).",
    "sniper_depthwise3x3_dgrad": "Data gradient of the depthwise convolution (depthwise_convolution-inl.h Backward, DepthwiseConv2dBackwardDataGpu), gather form.",
    "sniper_depthwise3x3_wgrad": "Weight gradient of the depthwise convolution (DepthwiseConv2dBackwardFilterGpu): dw[9,C] += per-channel correlation of dy with the shifted input; block partials summed in a fixed order through the slab of the stream's workspace (sniper_set_stream_workspace; bit-reproducible).",
    "sniper_im2col3x3s2_nchw": "im2col of MobileNetV2's first layer (3x3 / stride 2 / pad 1 over the 3-channel fp32 NCHW `data`, mobilenetv2_e2e.py:204-212) so that it runs on the wgmma GEMM; K order (kh, kw, ci), zero-padded to Kp.",
    "sniper_add_rows": "out = a + b on [M,C] rows: elemwise_add of the inverted-residual shortcut (mobilenetv2_e2e.py:22-24).",
    "sniper_relu_bwd": "dx = dy * (y > 0).",
    "sniper_maxpool3x3s2_nhwc": "Pooling max 3x3 stride 2 pad 1 (resnet_mx_101_e2e.py:409; nn/pool.cuh).",
    "sniper_stem_im2col": "im2col of bn_data(x) for conv0 (resnet_mx_101_e2e.py:402-404) so that the 7x7 stem runs on the wgmma kernel (sniper_gemm_nt with bn0 + ReLU as epilogue).",
    "sniper_stem_conv": "bn_data -> conv0 7x7/2 -> bn0 -> relu (resnet_mx_101_e2e.py:402-408), NCHW in, NHWC out.",
    "sniper_weight_transpose": "wt[ci, j, co] = w[co, sel[j], ci]: operand layout for data gradients.",
    "sniper_weight_transpose_batched": "Every sniper_weight_transpose of a training step in one launch (device job table).",
    "sniper_bn_param_grad_batched": "dgamma/dbeta of every BatchNorm in one launch (second half of sniper_bn_relu_bwd when it is called with dgamma = dbeta = NULL).",
    "sniper_colsum": "out[c] += sum_m x[m,c] (bias gradients; cudnnConvolutionBackwardBias).",
    "sniper_sgd_mom": "SGDMomKernel (optimizer_op-inl.h:279-300) on one flat buffer.",
    "sniper_sgd_mom_dev": "SGDMomKernel / MP_SGDMomKernel (optimizer_op-inl.h:279-300, 377-404) with lr and wd read from device memory, so that a captured CUDA graph follows WarmupMultiBatchScheduler (lib/train_utils/lr_scheduler.py:43-66); optional bf16 weight shadow = multi_precision.",
    "sniper_count_valid": "Device-side replacement of SoftmaxOutput's host valid count (softmax_output-inl.h:184-195).",
    "sniper_rpn_softmax_loss": "SoftmaxOutput(multi_output, use_ignore, normalization=valid) for the RPN (softmax_output-inl.h:108-132, 162-206): prob + gradient in one pass.",
    "sniper_rpn_smooth_l1_loss": "weight * smooth_l1(pred - target) + MakeLoss gradient for the RPN (mshadow_op.h:642-678; resnet_mx_101_e2e.py:330-334).",
    "sniper_softmax_ce": "SoftmaxOutput(normalization=valid, use_ignore) flat form (softmax_output-inl.h:207-263).",
    "sniper_smooth_l1_loss": "weight * smooth_l1(pred - target) + MakeLoss gradient (resnet_mx_101_e2e.py:318-319).",
    "sniper_deform_im2col": "deformable_im2col (contrib/nn/deformable_im2col.cuh:216-263), NHWC, whole batch.",
    "sniper_deform_col2im": "deformable_col2im + deformable_col2im_coord (contrib/nn/deformable_im2col.cuh:317-360, 419-480).",
    "sniper_deform_col2im_fp64acc": "sniper_deform_col2im with dx summed in a caller-owned fp64 scratch (reproducible run to run).",
    "sniper_anchor_target": "RPN anchor matching of anchor_worker.worker (lib/data_utils/data_workers.py:164-371) on device.",
    "sniper_focus_label": "FocusPixel labels of anchor_worker.worker's gen_mask (lib/data_utils/data_workers.py:165-192, TRAIN.AUTO_FOCUS) on device: the AutoFocus training label scale_label [B, Hf*Wf].",
    "sniper_focus_acc": "AutoFocusAccMetric (lib/train_utils/metric.py:50-72) on device: argmax hits and non-ignored pixels of the FocusPixel softmax, accumulated as exact float counts.",
    "sniper_soft_nms_batched":"cpu_soft_nms (lib/nms/cpu_nms.pyx:17-110; Gaussian / linear / hard) for every (image, class) problem of an inference scale in ONE launch: replaces the Pool(32) of nms_worker processes in Tester.aggregate (lib/inference.py:152-200). Same rows in the same order as the reference, exact score ties included (its row swaps are replayed); scratch: 24 bytes per row.",
    "sniper_proposal_nms_batched": "nmsp (lib/nms/nms.py:48-80, IoU threshold 0.7) of imdb.load_rpn_data (lib/dataset/imdb.py:81-118) for many images in ONE launch, one CTA per image: replaces the Pool(32) of host nmsp calls over the extracted RPN proposals. Keeps nmsp's float32 arithmetic and order; exact score ties go to the higher row.",
    "sniper_detect_post_workspace_bytes": "Scratch bytes for sniper_detect_post.",
    "sniper_detect_post": "Tester.detect's box decoding (lib/inference.py:100-139; nonlinear_pred lib/bbox/bbox_transform.py:93-133, clip_boxes, division by the scale), the score threshold and chip-border pruning of Tester.get_detections (lib/inference.py:232-351, check_valid :235-258) and the valid-range filter of Tester.aggregate (lib/inference.py:152-230, filter :176-186) for one batch of chips in ONE cooperative launch: surviving (x1, y1, x2, y2, score) rows appended to a caller-owned run buffer at a device-side cursor in (chip, roi, class) order, each with a 64-bit (image, class, scale, chip, roi) order key.  float64 decode, float32 rows rounded where the host path rounds them (no FMA).",
    "sniper_chip_input": "GPU input stage: im_worker.worker (lib/data_utils/data_workers.py:80-121) -- flip, cv2-style 8-bit bilinear resize by the chip scale, zero padding to crop_size, BGR->RGB minus PIXEL_MEANS -- from uint8 source rectangles to the fp32 NCHW `data` tensor of MNIteratorE2E (lib/iterators/MNIteratorE2E.py:194-199).",
    "sniper_chip_input_hw": "The same with a rectangular canvas: im_worker.worker_autofocus (lib/data_utils/data_workers.py:51-78) + the batch padding of MNIteratorTestAutoFocus._get_batch (lib/iterators/MNIteratorTestAutoFocus.py:36-78).",
    "sniper_anchor_subsample": "The npr.choice subsampling of anchor_worker.worker (data_workers.py:326-338) on device: <= num_fg positives, <= batch_size - #positives negatives per chip, the rest -> -1 (counter-based hash instead of numpy's RNG).",
    "sniper_anchor_subsample_at": "sniper_anchor_subsample for chips [chip_base, chip_base + B) of a larger batch (data_workers.py:326-338): chip b draws what chip chip_base + b of one launch over the whole batch draws, so each data-parallel rank subsamples its slice of the global batch (MNIteratorE2E with rank=) as the whole batch would; chip_base = 0 is sniper_anchor_subsample.",
    "sniper_chips_generate": "chips::cgenerate (lib/chips/cchips.cpp:54-177): host-side chip sampling, same rand() stream.",
    "sniper_chips_shuffle": "Host-only: the candidate orders of a sequence of sniper_chips_generate calls (std::random_shuffle over rand(), n_cand[c] - 1 draws per call; n_cand[c] = 0 is a call without boxes and draws nothing), written back to back to perm_out.  rand() ends where the calls would leave it.",
    "sniper_chip_plan_layout": "Host-only: fills the workspace column of a chip-plan table (the byte offset of each cover whose scratch does not fit in shared memory, -1 for the others) and the workspace size sniper_chip_plan_cover then needs.  The library never allocates the workspace.",
    "sniper_chip_plan_count": "The GT boxes chip_worker.chip_extractor (lib/data_utils/data_workers.py:394-450) selects for every (entry, scale) call of a chip-plan table in ONE launch: the integer size, fit and width / height tests of the host in float64.",
    "sniper_chip_plan_cover": "chips::cgenerate (lib/chips/cchips.cpp:54-177) for every (entry, scale) call of a chip-plan table in ONE launch, one block per call: mode 0 over the GT boxes chip_extractor selects (data_workers.py:394-450), mode 1 over the boxes no positive chip kept (box_assigner's negative chips, :540-594).  Boxes scaled and clipped as chip_generator does, the candidate order read from perm (sniper_chips_shuffle), the float32 containment test, the first-maximum greedy cover.  Writes each call's chips in pick order as float32 and divided by the scale in float64, and their count.  Bit-exact (no FMA).",
    "sniper_chip_plan_assign": "The box -> chip assignment of box_assigner (data_workers.py:452-594) for every call of a chip-plan table in ONE launch: owner = the first arg-max over the call's chips of the float64 ignore_overlaps (lib/bbox/bbox.pyx:59-95), kept iff the intersection is >= 1 on both sides and its sqrt-area in the scale's range (mode 0: positive chips, <= hi; mode 1: negative chips over the uncovered boxes, < hi).  owner_out int16 [boxes, S]: the owner, -1 selected but not kept, -2 not selected; left_count the selected boxes not kept.  Bit-exact (no FMA).",
    "sniper_cpu_nms": "cpu_nms (lib/nms/cpu_nms.pyx:112-163), host.",
    "sniper_cpu_soft_nms": "cpu_soft_nms (lib/nms/cpu_nms.pyx:17-110), host, in place.",
    "sniper_bbox_overlaps": "bbox_overlaps_cython / ignore_overlaps_cython (lib/bbox/bbox.pyx:17-95), host, float64.",
    "sniper_coco_box_iou_batched": "bbIou (lib/dataset/pycocotools/maskApi.c:98-109, reached through mask.iou from COCOeval.computeIoU, cocoeval.py:163-187) for every (category, image) pair of a CSR in ONE launch: pair p's [D_p x G_p] float64 matrix at out + iou_off[p]; crowd GTs (gt_flags bit 0) take the detection's area as the union.  Bit-exact (no FMA).",
    "sniper_coco_match": "COCOeval.evaluateImg (lib/dataset/pycocotools/cocoeval.py:189-272) for every pair x area range x IoU threshold in ONE launch: GTs ignore-sorted (stable), min(t, 1-1e-10), crowd re-matching, the stop at the first ignored GT, ties to the later GT, ids (not booleans) as the matched test.  Writes dt_flags[A,T,Dtot] (bit 0 matched, bit 1 ignored), npig[P,A] and gt_match[A,T,Gtot] (matching dt id, 0 = none, in ignore-sorted order); dt_match[A,T,Dtot] (matched gt id) and gt_order[A,Gtot] (ignore-sorted GT order) only when non-null.",
    "sniper_coco_accumulate": "COCOeval.accumulate (lib/dataset/pycocotools/cocoeval.py:274-374): precision[T,R,K,A,M] and recall[T,K,A,M] float64, one block per (category, area, maxDet, threshold), from sniper_coco_match's flags and one stable (category, descending score) order of the detections (cat_order) with their in-image ranks (dt_rank).  Byte-equal to the reference, -1 where it leaves -1.",
    "sniper_voc_match": "The matching loop of voc_eval (lib/dataset/pascal_voc_eval.py:137-171) for every (class, image) pair x overlap threshold in ONE launch, the pair's detections in the host's np.argsort(-confidence) order (:127-131): overlaps with +1 pixel extents, ovmax / jmax as np.max / np.argmax (a NaN wins, first maximum), the strict `ovmax > ovthresh`, difficult GTs neither tp nor fp, a second hit on a taken GT an fp.  flags[T,N] uint8: 1 tp, 2 fp, 0 neither; taken[T,G] is the reference's det scratch.  Bit-exact (no FMA).",
    "sniper_voc_accumulate": "pascal_voc_eval.py:173-179 and voc_ap (:39-70) for every class x threshold, one block each: integer tp / fp scans, rec = tp / float(npos), prec = tp / max(tp + fp, eps), then the 11-point AP (host recall thresholds, ap += p / 11. in order) or the area AP (mpre envelope, terms where mrec changes summed in numpy's pairwise order; terms is [T, N + C] scratch).  rec / prec [T,N] and ap [T,C] float64, byte-equal to the reference's.",
    "sniper_proposal_recall_workspace_bytes": "Host-only: per (area range, image) pair p = r * num_images + i, the byte offset of its IoU matrix in the workspace of sniper_proposal_recall_match (pair_ws_off_host[7 * num_images + 1]; pairs whose matrix fits in shared memory take none).  The workspace of pairs [b, e) is pair_ws_off[e] - pair_ws_off[b] bytes; the library never allocates it.",
    "sniper_proposal_recall_match": "The greedy matching of IMDB.evaluate_recall (lib/dataset/imdb.py:329-374) for pairs [pair_begin, pair_end) of (area range, image) in ONE launch, one block per pair: IoUs as bbox_overlaps_cython (lib/bbox/bbox.pyx:17-57) in float64 from uint16 / float32 / float64 proposals (prop_dtype 0 / 1 / 2) and float64 GTs; each round the best unused column maximum (argmax ties to the lower row, then the lower column), its row and column retired.  Writes each pair's round overlaps then zeros at gt_overlaps + pair_out_off[p]; status[p] = 1 where the reference asserts (best overlap < 0), 2 where bbox_overlaps_cython divides by zero.  Bit-exact (no FMA).",
    "sniper_proposal_recall_accumulate": "The statistics of IMDB.evaluate_recall (lib/dataset/imdb.py:307-328, 376-394) in ONE launch: counts[r * T + t] of gt_overlaps >= thresholds[t] per area range, then counts[7 * T + k] the proposals whose area (in their dtype) lies in range k + 1; recalls[r * T + t] = count / float(num_pos[r]), ar[r] = recalls.mean() in numpy's pairwise order, hist[k] = area_count / total_counts and hist[6] = total_counts / num_images.  counts / done are zeroed on the stream first.",
    "sniper_focus_chips_workspace_bytes": "Host-only: per FocusPixel map m of a sniper_focus_chips table, the byte offset of its scratch in the workspace (ws_off_host[n_maps + 1]; maps whose scratch fits in shared memory take none).  The library never allocates the workspace.",
    "sniper_focus_chips": "gmask of the AutoFocus inference (lib/chips/chips_inference.py:12-89) with the crop shift of add_chips (:91-173) for every FocusPixel map of a test scale in ONE launch, one block per map: the float32 threshold (mask >= float32 thresh), cv2.dilate with a d x d window anchored at d // 2, the contours of cv2.findContours(RETR_LIST) (outer borders of 8-connected foreground components, hole borders of 4-connected background regions that touch no frame row or column, listed by start pixel descending), _place with Python floor division, the merge loop until the contour count repeats (more than H * W + 2 passes: counts[m] = -1), then the scaling to image coordinates in double.  table: int64 [n_maps, 12] per map = address of its cell (0, 0) (float32), row and column strides in elements, H, W, iw, ih, then the float64 bits of im_width, im_height, cscale and the crop origin x, y.  Writes counts[m] chips of map m as float64 (x1, y1, x2, y2) at chips + (m * cap + k) * 4, the first cap of them (the caller re-launches maps with more); counts[m] = -2 when the table disagrees with table_host / ws_off.  Bit-exact (no FMA).",
    "sniper_train_metric_workspace_bytes": "Scratch bytes for sniper_train_metric_accum (zero-filled once by the caller; the kernel leaves it reusable).",
    "sniper_train_metric_accum": "The training metrics of lib/train_utils/metric.py:50-95, 104-300 (RPNAcc, RPNLogLoss, RPNL1Loss, RCNNAcc, RCNNLogLoss, RCNNL1LossCRCNN, AutoFocusAcc, AutoFocusLogLoss) for one step in ONE launch, added into a caller-owned accumulator (int64 num_inst[8] | int64 hits[8] | float64 sum[8]): replaces their per-step asnumpy() (:109-125).  Argmax ties to the first maximum, p + 1e-14 in float32, log and sums in float64, block partials summed in block order (byte-identical run to run).  num_inst from the step's count_valid results, the L1 sums from its loss buffer.",
    "sniper_nms_gpu":"Batched hard NMS on device for per-scale inference NMS (lib/nms/nms_kernel.cu:34-144 replacement).",
}


def signatures():
    out = []
    for f in sorted(glob.glob(os.path.join(ROOT, "sniper_b200", "csrc", "*.cu")) +
                    glob.glob(os.path.join(ROOT, "sniper_b200", "csrc", "*.cpp"))):
        s = open(f).read()
        for m in re.finditer(r'\n((?:int|size_t|const char\*)\s+(sniper_\w+)\s*\(([^)]*)\))\s*\{', s):
            out.append((os.path.basename(f), m.group(2), re.sub(r'\s+', ' ', re.sub(r'/\*.*?\*/', '', m.group(1)))))
    return out


def main():
    lines = ["/* sniper_b200 C-ABI -- generated by tools/gen_header.py from sniper_b200/csrc (do not edit by hand).",
             " *",
             " * Drop-in boundary of the SNIPER 512x512-chip training path: every entry point is extern \"C\", takes",
             " * plain pointers and sizes (device pointers unless a comment says host), a cudaStream_t passed as",
             " * void*, returns 0 on success and -1 on failure with the message in sniper_last_error().",
             " * No entry point allocates device memory or synchronises.  Reference file:line each one replaces",
             " * is cited above its prototype (paths relative to the reference repo; SNIPER-mxnet/src/operator/ is",
             " * implied for operator sources).",
             " */",
             "#ifndef SNIPER_B200_H_", "#define SNIPER_B200_H_", "#include <stddef.h>", "#include <stdint.h>", "",
             "#ifdef __cplusplus", 'extern "C" {', "#endif", ""]
    for f, name, sig in signatures():
        doc = DOC.get(name, "")
        lines.append("/* [%s] %s */" % (f, doc))
        lines.append(sig + ";")
        lines.append("")
    lines += ["#ifdef __cplusplus", "}", "#endif", "#endif  /* SNIPER_B200_H_ */", ""]
    os.makedirs(os.path.join(ROOT, "include"), exist_ok=True)
    open(os.path.join(ROOT, "include", "sniper_b200.h"), "w").write("\n".join(lines))


if __name__ == "__main__":
    main()
