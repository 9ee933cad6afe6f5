"""MobileNetV2 SNIPER training graph (BASELINE config 4) on the sm_90a kernels: NHWC, explicit backward.

Mirrors symbols/faster/mobilenetv2_e2e.py of the reference layer by layer, parameter names included:
  mobilenet_unit :27-43 (Convolution no_bias -> BatchNorm(momentum 0.995, eps 1e-5) -> clip(0, 6))
  inverted_residual_unit :46-90 (1x1 expand -> depthwise 3x3 -> 1x1 linear, elemwise_add shortcut)
  invresi_blocks :93-117, MNETV2_CONFIGS_MAP :120-135 (t, c, n, s)
  get_symbol_rcnn (is_train) :171-305: first-3x3-conv (stride 2), Cast(float16), 17 inverted residual units,
  last-1x1-conv (1280), Cast(float32), get_rpn :160-169 (256-d), conv_new_1, MultiProposalTarget (stride 32, 15
  anchors), DeformablePSROIPooling x2 (spatial_scale 1/32), fc_new_1/2 (512-d), cls_score / bbox_pred, losses with
  SoftmaxOutput(normalization='null') / (300 B) and MakeLoss / (188 B) (:281-296).
configs/faster/sniper_mobilenetv2_e2e.yml: FIXED_PARAMS = conv1, bn_conv1, res2.., gamma, beta -- of which only `gamma`
and `beta` match a MobileNetV2 parameter name: every convolution trains (the first one included), every BatchNorm runs
on batch statistics, its gamma / beta stay at their loaded values (registered here with lr_mult 0).

Where the work runs: the 1x1 expand / linear / last convolutions, the first layer (im2col + GEMM), the RPN / R-FCN head
and all their data / weight gradients on the wgmma kernel (gemm_tc.cu); the depthwise 3x3 layers, BatchNorm,
clip and the shortcut add are HBM-bound NHWC kernels (depthwise.cu, elementwise.cu).  The wgmma kernel moves operands
in 128-byte K atoms, so channel counts are zero-padded to multiples of 64 (16 / 24 / 32 -> 64, 96 -> 128, 144 / 160 ->
192): padded channels are exactly zero in the forward pass (zero weight rows, BatchNorm of a zero channel = beta = 0)
and receive exactly zero gradient (zero weight COLUMNS in the consumer), so the padded network computes the reference
network -- at 1.3-4x the memory traffic in the first three stages; a narrow-channel kernel for those stages is the
obvious next step (DESIGN.md).
Mixed precision (`Cfg.bf16`, the reference's TRAIN.fp16): bf16 activations / weight copies between the two Casts, fp32
BatchNorm arithmetic and statistics, fp32 (TF32) heads, fp32 master weights; bf16 has fp32's range, so TRAIN.scale = 1.
"""
import math

import numpy as np
import torch

from . import ops
from .model import Cfg, Conv, ParamStore, WgradScheduler, head_bwd, rfcn_detect, rfcn_fwd, rpn_train


def pad64(c):
    return (c + 63) // 64 * 64


class MCfg(Cfg):
    """The slice of configs/faster/sniper_mobilenetv2_e2e.yml the graph reads."""
    num_anchors = 15
    feat_stride = 32
    scales = (1, 2, 4, 8, 12)
    ratios = (0.5, 1, 2)
    batch_images = 40                 # BASELINE config 4: 320 chips on 8 GPUs (yml: 42)
    bn_eps = 1e-5
    bn_momentum = 0.995
    lr = 0.025
    warmup_step = 9000
    first_c = 32
    last_c = 1280
    bottlenecks = ((1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1))
    rpn_dim = 256
    fc_dim = 512
    first_kp = 64                     # 27 im2col columns padded to one K atom (64 bf16 / 2 x 32 fp32 elements)


ACT_NONE, ACT_RELU, ACT_RELU6 = 0, 1, 2          # affine_act codes; bn_act_bwd takes 3 for "none"


class MBN:
    """BatchNorm(fix_gamma=False, momentum=0.995, eps=1e-5) + optional clip(0, 6) on batch statistics."""

    def __init__(self, P, name, C, Cp, act):
        self.name, self.C, self.Cp, self.act = name, C, Cp, act
        self.P = P
        P.add(name + "_gamma", (Cp,), 0.0)          # FIXED_PARAMS: gamma / beta are not updated
        P.add(name + "_beta", (Cp,), 0.0)
        self.st = None

    def build(self, device, pool):
        P = self.P
        self.st = ops.BNState(self.Cp, device, P[self.name + "_gamma"], P[self.name + "_beta"],
                              P.grad(self.name + "_gamma"), P.grad(self.name + "_beta"), pool=pool)

    def fwd(self, x, cfg, have_stats=False, out=None):
        if have_stats:          # the producing GEMM's epilogue accumulated sum / sum of squares into st.sums
            ops.bn_finalize(self.st, x.numel() // self.Cp, eps=cfg.bn_eps, momentum=cfg.bn_momentum)
        else:
            ops.bn_stats(x, self.st, eps=cfg.bn_eps, momentum=cfg.bn_momentum)
        return ops.affine_act(x, self.st.scale, self.st.shift, relu=self.act, out=out)

    def bwd(self, x, dy, add=None):
        return ops.bn_act_bwd(x, dy, self.st, 3 if self.act == ACT_NONE else self.act, add=add, defer=True)


class Depthwise:
    """Convolution(kernel 3x3, pad 1, num_group = num_filter = C, no_bias): weights [9, Cp] fp32 (tap-major)."""

    def __init__(self, P, name, C, Cp, stride):
        self.name, self.C, self.Cp, self.stride = name, C, Cp, stride
        self.P = P
        P.add(name + "_weight", (9, Cp))

    @property
    def w(self):
        return self.P[self.name + "_weight"]

    def fwd(self, x):
        return ops.depthwise3x3(x, self.w, self.stride)

    def bwd_weight(self, dy, x):
        ops.depthwise3x3_wgrad(x, dy, self.P.grad(self.name + "_weight"), self.stride)

    def bwd_data(self, dy, in_hw):
        return ops.depthwise3x3_dgrad(dy, self.w, in_hw, self.stride)


class IRUnit:
    """inverted_residual_unit (mobilenetv2_e2e.py:46-90)."""

    def __init__(self, P, prefix, cin, cout, stride, t, shortcut, lowp):
        e = int(round(cin * t))
        self.prefix, self.cin, self.cout, self.e, self.stride, self.shortcut = prefix, cin, cout, e, stride, shortcut
        cinp, ep, coutp = pad64(cin), pad64(e), pad64(cout)
        self.exp = Conv(P, prefix + "-exp-conv2d", cinp, e, 1, cout_pad=ep, lowp=lowp)
        self.bn1 = MBN(P, prefix + "-exp-batchnorm", e, ep, ACT_RELU6)
        self.dw = Depthwise(P, prefix + "-depthwise-conv2d", e, ep, stride)
        self.bn2 = MBN(P, prefix + "-depthwise-batchnorm", e, ep, ACT_RELU6)
        self.lin = Conv(P, prefix + "-linear-conv2d", ep, cout, 1, cout_pad=coutp, lowp=lowp)
        self.bn3 = MBN(P, prefix + "-linear-batchnorm", cout, coutp, ACT_NONE)
        self.exp.cin_real, self.lin.cin_real = cin, e
        self.saved = None

    def convs(self):
        return [self.exp, self.lin]

    def bns(self):
        return [self.bn1, self.bn2, self.bn3]

    def fwd(self, x, cfg):
        c1 = self.exp.fwd(x, stats=self.bn1.st.sums)
        a1 = self.bn1.fwd(c1, cfg, have_stats=True)
        c2 = self.dw.fwd(a1)
        a2 = self.bn2.fwd(c2, cfg)
        c3 = self.lin.fwd(a2, stats=self.bn3.st.sums)
        y = self.bn3.fwd(c3, cfg, have_stats=True)
        if self.shortcut:
            ops.add_rows(y, x, out=y)
        self.saved = (x, c1, a1, c2, a2, c3)
        return y

    def bwd(self, dy, cfg, need_dx=True):
        x, c1, a1, c2, a2, c3 = self.saved
        W = cfg.wsched
        sp = cfg.wgrad_splits
        hw_in = (x.shape[1], x.shape[2])
        hw_mid = (c2.shape[1], c2.shape[2])
        dc3 = self.bn3.bwd(c3, dy)
        W(self.lin.bwd_weight, dc3, a2, sp)
        da2 = self.lin.bwd_data(dc3, hw_mid)
        dc2 = self.bn2.bwd(c2, da2)
        W(self.dw.bwd_weight, dc2, a1)
        da1 = self.dw.bwd_data(dc2, hw_in)
        dc1 = self.bn1.bwd(c1, da1)
        W(self.exp.bwd_weight, dc1, x, sp)
        self.saved = None
        if not need_dx:
            return None
        return self.exp.bwd_data(dc1, hw_in, residual=dy if self.shortcut else None)


class SniperMobileNetV2:
    """mobilenetv2_e2e.get_symbol_rcnn(cfg, is_train=True) as an executable object."""

    n_phases = 1
    # the R-CNN loss is not normalised by the valid count (:281-282), so cnt_buf[1] stays 0: the trainer's metric
    # launch counts the rows itself
    rcnn_valid_counted = False
    af = None                         # the reference's MobileNetV2 graph has no FocusPixel branch (tester.DetectionNetwork)

    @property
    def feat_stride(self):
        return self.cfg.feat_stride

    def __init__(self, cfg=None, device="cuda", seed=5):
        self.cfg = cfg or MCfg()
        cfg = self.cfg
        self.device = device
        cfg.wsched = WgradScheduler(bool(cfg.wgrad_stream))
        lowp = bool(cfg.bf16)
        self.act_dtype = torch.bfloat16 if lowp else torch.float32
        P = self.P = ParamStore()
        P.bucket = 0
        fc, fcp = cfg.first_c, pad64(cfg.first_c)
        self.first = Conv(P, "first-3x3-conv-conv2d", cfg.first_kp, fc, 1, cout_pad=fcp, need_dgrad=False, lowp=lowp)
        self.first.cin_real = 27
        self.bn_first = MBN(P, "first-3x3-conv-batchnorm", fc, fcp, ACT_RELU6)
        self.units = []
        in_c = fc
        for i, (t, c, n, s) in enumerate(cfg.bottlenecks):
            for j in range(n):
                self.units.append(IRUnit(P, "seq-%d-block%d" % (i, j), in_c if j == 0 else c, c, s if j == 0 else 1, t,
                                         shortcut=(j > 0), lowp=lowp))
            in_c = c
        self.last = Conv(P, "last-1x1-conv-conv2d", pad64(in_c), cfg.last_c, 1, lowp=lowp)
        self.last.cin_real = in_c
        self.bn_last = MBN(P, "last-1x1-conv-batchnorm", cfg.last_c, cfg.last_c, ACT_RELU6)
        A, D = cfg.num_anchors, cfg.last_c
        self.rpn_conv = Conv(P, "rpn_conv_3x3", D, cfg.rpn_dim, 3, 1, 1, 1, bias=True)
        # rpn_bbox_pred (4A) and rpn_cls_score (2A) fused into one 1x1 conv: rows [0,4A) | [4A,6A), padded to 96
        self.rpn_head = Conv(P, "rpn_head", cfg.rpn_dim, 6 * A, 1, bias=True, cout_pad=(6 * A + 31) // 32 * 32)
        self.conv_new_1 = Conv(P, "conv_new_1", D, 256, 1, bias=True)
        self.fc_offset = Conv(P, "offset", 7 * 7 * 256, 98, 1, bias=True, cout_pad=128, lr_mult=0.01)
        self.fc_new_1 = Conv(P, "fc_new_1", 7 * 7 * 256, cfg.fc_dim, 1, bias=True)
        self.fc_new_2 = Conv(P, "fc_new_2", cfg.fc_dim, cfg.fc_dim, 1, bias=True)
        self.fc_out = Conv(P, "cls_bbox", cfg.fc_dim, cfg.num_classes + 4, 1, bias=True, cout_pad=96)
        P.finalize(device, lowp=lowp)
        self._init_weights(seed)
        self.loss_buf = torch.zeros(8, device=device)
        self.cnt_buf = torch.zeros(2, dtype=torch.int32, device=device)
        self._wt_table = None
        self._bn_table = None
        self.step_count = 0

    # ---------------------------------------------------------------- parameters
    def backbone_convs(self):
        return [self.first] + [c for u in self.units for c in u.convs()] + [self.last]

    def head_convs(self):
        return [self.rpn_conv, self.rpn_head, self.conv_new_1, self.fc_offset, self.fc_new_1, self.fc_new_2, self.fc_out]

    def all_bns(self):
        return [self.bn_first] + [b for u in self.units for b in u.bns()] + [self.bn_last]

    train_bns = all_bns

    def _init_weights(self, seed):
        """He-normal backbone over the REAL fan-in, N(0, 0.01) heads, zero offset FC (init_weight_rcnn :364-391); one
        host image of the parameter buffer, one H2D.  Padded rows AND columns are zero (see the module docstring)."""
        cfg, P, dev = self.cfg, self.P, self.device
        g = torch.Generator()
        g.manual_seed(seed)
        host = torch.zeros(P.total)

        def put(name, t):
            o, shape = P.layout[name]
            assert tuple(t.shape) == tuple(shape), (name, t.shape, shape)
            host[o:o + t.numel()] = t.reshape(-1)

        for c in self.backbone_convs():
            w = torch.zeros(c.coutp, c.K)
            w[:c.cout, :c.cin_real].normal_(0, math.sqrt(2.0 / c.cin_real), generator=g)
            put(c.name + "_weight", w)
        for u in self.units:
            w = torch.zeros(9, u.dw.Cp)
            w[:, :u.dw.C].normal_(0, math.sqrt(2.0 / 9.0), generator=g)
            put(u.dw.name + "_weight", w)
        for c in self.head_convs():
            w = torch.zeros(c.coutp, c.K)
            if c is not self.fc_offset:
                w[:c.cout].normal_(0, 0.01, generator=g)
            put(c.name + "_weight", w)
        bns = self.all_bns()
        pool = ops.BNPool(sum(b.Cp for b in bns), dev)
        for b in bns:
            b.build(dev, pool)
            o, _ = P.layout[b.name + "_gamma"]
            host[o:o + b.Cp] = 1.0
        P.w.copy_(host)
        P.sync_lowp()
        pool.finalize()
        self.bn_pool = pool

    # ---------------------------------------------------------------- one training step
    def forward_backward(self, batch, on_bucket=None):
        out = None
        for k, out in enumerate(self.fb_phases(batch)):
            if on_bucket is not None:
                on_bucket(k)
        return out

    def fb_phases(self, batch):
        """One forward + backward pass (a single gradient bucket: one `yield`).  batch: the tensors of MNIteratorE2E for
        this configuration -- data [B,3,512,512], label [B, 15*16*16], bbox_target / bbox_weight [B,60,16,16], gt_boxes
        [B,100,5], valid_ranges [B,2], im_info [B,3] (`crowd_boxes` of the symbol is not read by the operator)."""
        cfg, P = self.cfg, self.P
        data = batch["data"]
        dev = data.device
        lowp = bool(cfg.bf16)
        P.g.zero_()
        self.loss_buf.zero_()
        self.cnt_buf.zero_()
        if self._wt_table is None:
            jobs = [j for c in self.backbone_convs() + self.head_convs() for j in c.bwd_jobs()]
            self._wt_table = ops.weight_transpose_jobs(jobs, dev)
            self._bn_table = ops.bn_param_grad_jobs([b.st for b in self.all_bns()], dev)
        ops.weight_transpose_batched(self._wt_table)

        # ---- backbone forward
        col = ops.im2col3x3s2(data, cfg.first_kp, dtype=self.act_dtype)              # [B,256,256,64]
        c0 = self.first.fwd(col, stats=self.bn_first.st.sums)
        x = self.bn_first.fwd(c0, cfg, have_stats=True)                               # the reference's Cast sits here
        a0 = x
        for u in self.units:
            x = u.fwd(x, cfg)
        cl = self.last.fwd(x, stats=self.bn_last.st.sums)
        al = self.bn_last.fwd(cl, cfg, have_stats=True)
        feat_in = ops.cast_rows(al, torch.float32) if lowp else al                    # Cast(float32) (:226)

        # ---- RPN (get_rpn) + conv_new_1
        rpn = self.rpn_conv.fwd(feat_in, relu=True)
        head = self.rpn_head.fwd(rpn)                                     # [B,H,W,96]: 4A deltas | 2A scores
        feat = self.conv_new_1.fwd(feat_in, relu=True)
        prob, dhead, rois, label, bbox_target, bbox_weight = rpn_train(self, batch, head)
        N = rois.shape[0]
        out, rfcn = rfcn_fwd(self, feat, rois)                                                     # [N,96]
        K = cfg.num_classes
        dout = torch.zeros_like(out)
        cls_prob = torch.empty(N, K, device=dev)
        # SoftmaxOutput without normalization (:281-282): gradient (p - onehot) * grad_scale / (300 B), ignore rows 0
        ops.softmax_ce(out, label, K, cfg.grad_scale / (300.0 * cfg.batch_images), None, cls_prob, dout,
                       self.loss_buf[2:3])
        ops.smooth_l1_loss(out[:, K:K + 4], bbox_target, bbox_weight, 4, cfg.grad_scale / (188.0 * cfg.batch_images),
                           dout[:, K:K + 4], self.loss_buf[3:4])

        # ================= backward =================
        sp = cfg.wgrad_splits
        W = cfg.wsched
        dfi = head_bwd(self, feat_in, rpn, dhead, dout, rfcn)
        g = ops.cast_rows(dfi, torch.bfloat16) if lowp else dfi                  # backward of the Cast
        # ---- backbone backward
        dcl = self.bn_last.bwd(cl, g)
        W(self.last.bwd_weight, dcl, x, sp)
        g = self.last.bwd_data(dcl, (x.shape[1], x.shape[2]))
        for u in reversed(self.units):
            g = u.bwd(g, cfg)
        dc0 = self.bn_first.bwd(c0, g)
        W(self.first.bwd_weight, dc0, col, sp)
        ops.bn_param_grad_batched(self._bn_table)
        W.join()
        self.step_count += 1
        yield dict(rpn_cls_prob=prob, rpn_bbox_loss=self.loss_buf[1:2], cls_prob=cls_prob, bbox_loss=self.loss_buf[3:4],
                   label=label, rois=rois, losses=self.loss_buf, rpn_head=head, last_fm=feat_in, first=a0,
                   bbox_target=bbox_target, bbox_weight=bbox_weight)

    # ---------------------------------------------------------------- inference graph
    def forward_inference(self, data, im_info, rpn_pre_nms_top_n=6000, autofocus=False):
        """mobilenetv2_e2e.get_symbol_rcnn(cfg, is_train=False) (:306-362): every BatchNorm on its moving statistics,
        SoftmaxActivation over the RPN scores, MultiProposal (TEST.RPN_PRE_NMS_TOP_N 6000, 300 rois per image, stride 32),
        deformable R-FCN head -> (rois [B*R,5], rpn scores [B*R], cls_prob [B*R,K], bbox_pred [B*R,4]).  No parameter is
        touched.  BatchNorm + clip run as one `sniper_affine_act` pass per layer (the GEMM epilogue has ReLU, not clip).
        autofocus: the `tester.DetectionNetwork` argument; this graph has no FocusPixel branch, so True is refused."""
        if autofocus:
            raise RuntimeError("forward_inference(autofocus=True): the MobileNetV2 graph has no FocusPixel branch")
        cfg = self.cfg
        lowp = bool(cfg.bf16)
        for b in self.all_bns():
            ops.bn_frozen(b.st, cfg.bn_eps)            # scale / shift from the moving statistics (the next training
        act = lambda bn, t: ops.affine_act(t, bn.st.scale, bn.st.shift, relu=bn.act)    # step recomputes them)
        col = ops.im2col3x3s2(data, cfg.first_kp, dtype=self.act_dtype)
        x = act(self.bn_first, self.first.fwd(col))
        for u in self.units:
            a1 = act(u.bn1, u.exp.fwd(x))
            a2 = act(u.bn2, u.dw.fwd(a1))
            y = act(u.bn3, u.lin.fwd(a2))
            if u.shortcut:
                ops.add_rows(y, x, out=y)
            x = y
        al = act(self.bn_last, self.last.fwd(x))
        feat_in = ops.cast_rows(al, torch.float32) if lowp else al
        rpn = self.rpn_conv.fwd(feat_in, relu=True)
        head = self.rpn_head.fwd(rpn)
        feat = self.conv_new_1.fwd(feat_in, relu=True)
        return rfcn_detect(self, head, feat, im_info, rpn_pre_nms_top_n=rpn_pre_nms_top_n)

    # ---------------------------------------------------------------- optimizer
    def set_lr(self, lr=None):
        self.P.set_hyper(float(self.cfg.lr if lr is None else lr), float(self.cfg.wd))

    def update(self, lr=None):
        if lr is not None or self.P._hyper_host[0] is None:
            self.set_lr(lr)
        self.P.sgd_step(self.cfg.momentum)

    def train_step(self, batch, lr=None, allreduce=None):
        out = self.forward_backward(batch)
        if allreduce is not None:
            allreduce(self.P.g)
        self.update(lr)
        return out

    # ---------------------------------------------------------------- reference checkpoints (names / layouts of the symbol)
    def export_reference(self, grads=False):
        """(arg_params, aux_params) under the reference's names and layouts -- OIHW convolutions incl. the (C,1,3,3)
        depthwise filters, real channel counts (padding stripped); grads=True: the parameter gradients of the last
        forward_backward instead (BatchNorm gamma / beta are fixed parameters: no gradient entries, as in the reference)."""
        from . import checkpoint as ck
        cfg = self.cfg
        A, K = cfg.num_anchors, cfg.num_classes
        n = lambda t: t.detach().cpu().numpy().copy()
        src = (lambda name: self.P.grad(name)) if grads else (lambda name: self.P[name])
        arg, aux = {}, {}
        w = n(src(self.first.name + "_weight"))[:cfg.first_c, :27]
        arg[self.first.name + "_weight"] = np.ascontiguousarray(w.reshape(cfg.first_c, 3, 3, 3).transpose(0, 3, 1, 2))
        for c in self.backbone_convs()[1:]:
            w = n(src(c.name + "_weight"))[:c.cout, :c.cin_real]
            arg[c.name + "_weight"] = np.ascontiguousarray(w.reshape(c.cout, c.cin_real, 1, 1))
        for u in self.units:
            w = n(src(u.dw.name + "_weight"))[:, :u.dw.C]
            arg[u.dw.name + "_weight"] = np.ascontiguousarray(w.T.reshape(u.dw.C, 1, 3, 3))
        parts = {"rpn_head": (4 * A, 2 * A), "cls_bbox": (K, 4)}
        for c in self.head_convs():
            b = n(src(c.name + "_bias"))
            ck.conv_to_reference(c.name, c.cout, c.cin, c.k, n(src(c.name + "_weight")), b, parts.get(c.name), arg)
        if not grads:
            for bn in self.all_bns():
                arg[bn.name + "_gamma"] = n(bn.st.gamma)[:bn.C]
                arg[bn.name + "_beta"] = n(bn.st.beta)[:bn.C]
                aux[bn.name + "_moving_mean"] = n(bn.st.moving_mean)[:bn.C]
                aux[bn.name + "_moving_var"] = n(bn.st.moving_var)[:bn.C]
        return arg, aux

    def load_reference(self, arg, aux):
        """The inverse of export_reference: a reference checkpoint (numpy dicts) into the padded layouts."""
        from . import checkpoint as ck
        cfg, dev = self.cfg, self.device
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
        w = np.zeros((self.first.coutp, self.first.K), np.float32)
        w[:cfg.first_c, :27] = np.asarray(arg[self.first.name + "_weight"]).transpose(0, 2, 3, 1).reshape(cfg.first_c, 27)
        self.first.master.copy_(t(w))
        for c in self.backbone_convs()[1:]:
            w = np.zeros((c.coutp, c.K), np.float32)
            w[:c.cout, :c.cin_real] = np.asarray(arg[c.name + "_weight"]).reshape(c.cout, c.cin_real)
            c.master.copy_(t(w))
        for u in self.units:
            w = np.zeros((9, u.dw.Cp), np.float32)
            w[:, :u.dw.C] = np.asarray(arg[u.dw.name + "_weight"]).reshape(u.dw.C, 9).T
            u.dw.w.copy_(t(w))
        for c in self.head_convs():
            w, b = ck.conv_from_reference(c.name, c.cout, c.coutp, c.cin, c.k, True, arg)
            c.master.copy_(t(w))
            c.b.copy_(t(b))
        for bn in self.all_bns():
            for dst, v, fill in ((bn.st.gamma, arg[bn.name + "_gamma"], 1.0), (bn.st.beta, arg[bn.name + "_beta"], 0.0),
                                 (bn.st.moving_mean, aux[bn.name + "_moving_mean"], 0.0),
                                 (bn.st.moving_var, aux[bn.name + "_moving_var"], 1.0)):
                full = np.full((bn.Cp,), fill, np.float32)
                full[:bn.C] = np.asarray(v)
                dst.copy_(t(full))
        self.P.sync_lowp()
        self._wt_table = None
