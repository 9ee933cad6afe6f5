"""Float64 references of deformable convolution (csrc/deform_conv.cu) and (Deformable)PSROIPooling (csrc/psroi.cu).

Sample geometry -- every position, floor / ceil, clamp and validity test -- is evaluated in float32 torch ops in the
kernels' operation order (one correctly rounded torch op per kernel op, never fused), so it reproduces the kernels'
indices and fractional parts exactly.  Everything downstream of the geometry is float64: the bilinear values, sums, means
and the data / offset / trans gradients, written out as explicit formulas.  Weights come in two variants: the exact
float64 products of the float32 fractions ("exact"), and the kernels' own float32 weights ("kernel": fl(1-lh), fl(hh*hw),
...), so that where a kernel's only rounding is its final sum the comparison can be held to about one ulp.

Alongside each result the functions return the float64 sum of the absolute values of its terms (the scale of any
rounding error) and, for scattered gradients, the number of terms each element receives (the length of the chain of
atomic additions that forms it).  Everything is vectorised torch and runs on whatever device its inputs are on; the
large gathers are done in chunks of rois / images."""
import torch

F32, F64 = torch.float32, torch.float64
CHUNK = 1 << 26            # elements of the largest float64 gather held at a time


def _round_away(x):
    """roundf: nearest integer, ties away from zero (torch.round rounds ties to even).  |x| + 0.5 is exact in float64
    for any float32 x, so the floor is the correctly rounded result."""
    x64 = x.double()
    return (torch.sign(x64) * torch.floor(x64.abs() + 0.5)).to(F32)


# ----------------------------------------------------------------------------------------------- deformable conv


def out_extent(extent, k, stride, dil, pad):
    span = extent + 2 * pad - dil * (k - 1) - 1
    return 0 if span < 0 else span // stride + 1


def dc_geom(offset, H, W, KH, KW, stride, dil, pad, dgroups):
    """make_sample of deform_conv.cu for every (n, ho, wo, group, tap).  offset: float32 [NB, Ho, Wo, off_ld] with
    channel g*2*KK + 2*tap + {0: dh, 1: dw}.  Returns dict of [NB, Ho, Wo, dg, KK] tensors: valid, absolute corner rows /
    columns hl, hh, wl, wh (int64) and the float32 fractions lh, lw."""
    NB, Ho, Wo, _ = offset.shape
    dev = offset.device
    KK = KH * KW
    off = offset[..., :dgroups * 2 * KK].reshape(NB, Ho, Wo, dgroups, KK, 2)
    off_h, off_w = off[..., 0], off[..., 1]
    tap = torch.arange(KK, device=dev)
    idil = ((tap // KW) * dil).view(1, 1, 1, 1, KK)
    jdil = ((tap % KW) * dil).view(1, 1, 1, 1, KK)
    h_in = (torch.arange(Ho, device=dev) * stride - pad).view(1, Ho, 1, 1, 1)
    w_in = (torch.arange(Wo, device=dev) * stride - pad).view(1, 1, Wo, 1, 1)
    h_im = (h_in + idil).to(F32) + off_h
    w_im = (w_in + jdil).to(F32) + off_w
    valid = (h_im >= 0) & (w_im >= 0) & (h_im < H) & (w_im < W)

    def axis(rel, o, base, extent):
        m = rel.to(F32) + o
        cur = extent - base
        low = torch.floor(m)
        clamp = low >= (cur - 1).to(F32)
        lo = torch.where(clamp, (cur - 1).expand_as(low), low.long())
        hi = torch.where(clamp, lo, lo + 1)
        m = torch.where(clamp, lo.to(F32), m)
        frac = m - lo.to(F32)
        return base + lo, base + hi, frac

    hl, hh, lh = axis(idil, off_h, h_in, H)
    wl, wh, lw = axis(jdil, off_w, w_in, W)
    return dict(valid=valid, hl=hl, hh=hh, wl=wl, wh=wh, lh=lh, lw=lw)


def dc_weights(g, kind):
    """The four bilinear weights (float64) of corners (hl,wl), (hl,wh), (hh,wl), (hh,wh); zero for invalid samples."""
    lh, lw = g["lh"], g["lw"]
    if kind == "exact":
        lh, lw = lh.double(), lw.double()
        ws = [(1 - lh) * (1 - lw), (1 - lh) * lw, lh * (1 - lw), lh * lw]
    else:
        hh, hw = 1 - lh, 1 - lw                       # float32, as the kernel
        ws = [(hh * hw).double(), (hh * lw).double(), (lh * hw).double(), (lh * lw).double()]
    v = g["valid"].double()
    return [w * v for w in ws]


def _corners(g):
    return [(g["hl"], g["wl"]), (g["hl"], g["wh"]), (g["hh"], g["wl"]), (g["hh"], g["wh"])]


def _img_chunks(NB, per_image):
    step = max(1, CHUNK // max(1, per_image))
    return [(s, min(NB, s + step)) for s in range(0, NB, step)]


def _gather(x, n0, n1, y, xx, c0, c1):
    """x[n, y, x, c0:c1] for the [n1-n0, Ho, Wo, KK] index tensors y / xx (clamped: invalid samples carry weight 0)"""
    H, W = x.shape[1], x.shape[2]
    nidx = torch.arange(n0, n1, device=x.device).view(-1, 1, 1, 1)
    return x[nidx, y.clamp(0, H - 1), xx.clamp(0, W - 1), c0:c1]


def dc_im2col(x, offset, KH, KW, stride, dil, pad, dgroups, kind="exact"):
    """col [NB*Ho*Wo, KK*C] (tap-major) in float64 and the sum of |w_q * x_q| per element.  x: [NB,H,W,C] (any float
    dtype; the stored values are used), offset: float32 [NB,Ho,Wo,off_ld]."""
    NB, H, W, C = x.shape
    KK = KH * KW
    cpg = C // dgroups
    Ho, Wo = offset.shape[1], offset.shape[2]
    x = x.double()
    col = torch.empty(NB, Ho, Wo, KK, C, dtype=F64, device=x.device)
    mag = torch.empty_like(col)
    for n0, n1 in _img_chunks(NB, Ho * Wo * KK * C * 4):
        g = dc_geom(offset[n0:n1], H, W, KH, KW, stride, dil, pad, dgroups)
        ws = dc_weights(g, kind)
        for d in range(dgroups):
            c0, c1 = d * cpg, (d + 1) * cpg
            acc = 0
            am = 0
            for w, (yy, xx) in zip(ws, _corners(g)):
                v = _gather(x, n0, n1, yy[..., d, :], xx[..., d, :], c0, c1)
                t = w[..., d, :, None] * v
                acc = acc + t
                am = am + t.abs()
            col[n0:n1, ..., c0:c1] = acc
            mag[n0:n1, ..., c0:c1] = am
    return col.view(NB * Ho * Wo, KK * C), mag.view(NB * Ho * Wo, KK * C)


def dc_col2im(dcol, x, offset, KH, KW, stride, dil, pad, dgroups, kind="exact"):
    """Transposes of dc_im2col in float64: returns dict(dx, dx_mag, dx_terms, doff, doff_mag).
    dx [NB,H,W,C]: sum over samples of w_q * dcol (dx_mag: of |w_q * dcol|; dx_terms: number of non-zero-weight
    contributions per element).  doff [NB,Ho,Wo,dg*2*KK] in the offset layout: d/dh and d/dw of sum(col * dcol), i.e.
    sum_c dcol * ((1-lw)(v3-v1) + lw(v4-v2)) and sum_c dcol * ((1-lh)(v2-v1) + lh(v4-v3)) for valid samples, 0 else."""
    NB, H, W, C = x.shape
    KK = KH * KW
    cpg = C // dgroups
    Ho, Wo = offset.shape[1], offset.shape[2]
    xd = x.double()
    dc = dcol.double().view(NB, Ho, Wo, KK, C)
    dev = x.device
    dx = torch.zeros(dgroups, NB * H * W, cpg, dtype=F64, device=dev)
    dxm = torch.zeros_like(dx)
    dxt = torch.zeros(dgroups, NB * H * W, dtype=F64, device=dev)
    doff = torch.zeros(NB, Ho, Wo, dgroups, KK, 2, dtype=F64, device=dev)
    doffm = torch.zeros_like(doff)
    for n0, n1 in _img_chunks(NB, Ho * Wo * KK * C * 4):
        g = dc_geom(offset[n0:n1], H, W, KH, KW, stride, dil, pad, dgroups)
        ws = dc_weights(g, kind)
        valid = g["valid"].double()
        lh, lw = g["lh"].double(), g["lw"].double()
        nidx = torch.arange(n0, n1, device=dev).view(-1, 1, 1, 1)
        for d in range(dgroups):
            c0, c1 = d * cpg, (d + 1) * cpg
            gc = dc[n0:n1, ..., c0:c1]
            vs = []
            for w, (yy, xx) in zip(ws, _corners(g)):
                yy, xx = yy[..., d, :], xx[..., d, :]
                vs.append(_gather(xd, n0, n1, yy, xx, c0, c1))
                wq = w[..., d, :]
                flat = ((nidx * H + yy.clamp(0, H - 1)) * W + xx.clamp(0, W - 1)).reshape(-1)
                t = wq[..., None] * gc
                dx[d].index_add_(0, flat, t.reshape(-1, cpg))
                dxm[d].index_add_(0, flat, t.abs().reshape(-1, cpg))
                dxt[d].index_add_(0, flat, (wq != 0).double().reshape(-1))
            v1, v2, v3, v4 = vs
            vd = valid[..., d, :, None]
            fh, fw = lh[..., d, :, None], lw[..., d, :, None]
            dh = gc * ((1 - fw) * (v3 - v1) + fw * (v4 - v2)) * vd
            dw = gc * ((1 - fh) * (v2 - v1) + fh * (v4 - v3)) * vd
            dhm = gc.abs() * ((1 - fw) * (v3.abs() + v1.abs()) + fw * (v4.abs() + v2.abs())) * vd
            dwm = gc.abs() * ((1 - fh) * (v2.abs() + v1.abs()) + fh * (v4.abs() + v3.abs())) * vd
            doff[n0:n1, :, :, d, :, 0] = dh.sum(-1)
            doff[n0:n1, :, :, d, :, 1] = dw.sum(-1)
            doffm[n0:n1, :, :, d, :, 0] = dhm.sum(-1)
            doffm[n0:n1, :, :, d, :, 1] = dwm.sum(-1)
    per_c = lambda t: t.permute(1, 0, 2).reshape(NB, H, W, C)
    return dict(dx=per_c(dx), dx_mag=per_c(dxm),
                dx_terms=dxt.t().reshape(NB, H, W, dgroups).repeat_interleave(cpg, -1),
                doff=doff.view(NB, Ho, Wo, -1), doff_mag=doffm.view(NB, Ho, Wo, -1))


# ----------------------------------------------------------------------------------------------- (deformable) PSROI


def ps_geom(rois, trans, *, H, W, spatial_scale, pooled, part_size, sample_per_part, trans_std, no_trans, ncls):
    """deform_geom + sample_pos of psroi.cu for every (roi, class, ph / pw, sample).  rois float32 [N,5], trans float32
    [N, 2*ncls, part, part] or None.  The sample grid of a bin is separable: the column of sample (ih, iw) depends on iw
    only, its row on ih only, and a sample is taken iff both are inside, so the per-axis tables below describe every
    sample.  Returns a dict; x-axis tensors are [N, ncls, P(ph), P(pw), S], y-axis ones the same with S over ih."""
    dev = rois.device
    N, P, S = rois.shape[0], pooled, sample_per_part
    part = part_size or pooled
    f = lambda v: torch.tensor(v, dtype=F32, device=dev)
    sc = f(spatial_scale)
    b = rois[:, 0].long()
    r = _round_away(rois[:, 1:5])
    start_w = ((r[:, 0] * sc).double() - 0.5).to(F32)
    start_h = ((r[:, 1] * sc).double() - 0.5).to(F32)
    end_w = ((((r[:, 2].double() + 1.0).to(F32)) * sc).double() - 0.5).to(F32)
    end_h = ((((r[:, 3].double() + 1.0).to(F32)) * sc).double() - 0.5).to(F32)
    roi_w = torch.clamp((end_w - start_w).double(), min=0.1).to(F32)
    roi_h = torch.clamp((end_h - start_h).double(), min=0.1).to(F32)
    bin_w, bin_h = roi_w / f(P), roi_h / f(P)
    sub_w, sub_h = bin_w / f(S), bin_h / f(S)
    pidx = torch.arange(P, device=dev)
    part_idx = torch.floor((pidx.to(F32) / f(P)) * f(part)).long()                 # part_h of ph / part_w of pw
    if no_trans:
        tx = torch.zeros(N, ncls, P, P, dtype=F32, device=dev)
        ty = torch.zeros_like(tx)
    else:
        t = trans.view(N, ncls, 2, part, part)
        ph_, pw_ = part_idx.view(P, 1), part_idx.view(1, P)
        tx = t[:, :, 0][:, :, ph_, pw_] * f(trans_std)                            # [N, ncls, P(ph), P(pw)]
        ty = t[:, :, 1][:, :, ph_, pw_] * f(trans_std)
    pf = pidx.to(F32)
    wstart = (pf.view(1, 1, 1, P) * bin_w.view(N, 1, 1, 1)) + start_w.view(N, 1, 1, 1)
    wstart = wstart + tx * roi_w.view(N, 1, 1, 1)
    hstart = (pf.view(1, 1, P, 1) * bin_h.view(N, 1, 1, 1)) + start_h.view(N, 1, 1, 1)
    hstart = hstart + ty * roi_h.view(N, 1, 1, 1)
    sf = torch.arange(S, device=dev).to(F32)

    def axis(start, sub, extent):
        c = start[..., None] + sf * sub.view(N, 1, 1, 1, 1)
        c64 = c.double()
        ok = (c64 >= -0.5) & (c64 <= extent - 0.5)
        c = torch.clamp(c64, 0.0, extent - 1.0).to(F32)
        lo, hi = torch.floor(c), torch.ceil(c)
        return dict(pos=c, ok=ok, lo=lo.long(), hi=hi.long(), dist=c - lo)

    return dict(b=b, roi_w=roi_w, roi_h=roi_h, part_idx=part_idx, x=axis(wstart, sub_w, W), y=axis(hstart, sub_h, H),
                N=N, P=P, S=S, ncls=ncls, part=part)


def ps_count(g):
    """valid samples per bin [N, ncls, P, P] (what the kernels divide by)"""
    return g["y"]["ok"].sum(-1) * g["x"]["ok"].sum(-1)


def ps_sample_idx(g, W, output_dim, channels_each_class):
    """oracle_deform_psroi_fwd's sample_idx [N*output_dim*P*P, S*S, 4] (NCHW order; -1 for a skipped sample)"""
    N, P, S = g["N"], g["P"], g["S"]
    y, x = g["y"], g["x"]
    # [N, ncls, P, P, S(ih), S(iw)]
    y1, y2 = y["lo"][..., :, None], y["hi"][..., :, None]
    x1, x2 = x["lo"][..., None, :], x["hi"][..., None, :]
    ok = y["ok"][..., :, None] & x["ok"][..., None, :]
    idx = torch.stack(torch.broadcast_tensors(y1 * W + x1, y2 * W + x1, y1 * W + x2, y2 * W + x2), -1)
    idx = torch.where(ok[..., None], idx, torch.full_like(idx, -1))
    cls = torch.arange(output_dim, device=idx.device) // channels_each_class
    return idx[:, cls].reshape(N * output_dim * P * P, S * S, 4).int()


def _axis_tab(a, kind):
    """per-axis (index, weight, d weight / d coordinate) of the 2S corner entries [.., 2S]: entry 2s is the low
    corner of sample s, 2s + 1 its high corner; invalid samples get weight 0"""
    ok = a["ok"].double()
    dist = a["dist"]
    if kind == "exact":
        wlo, whi = 1 - dist.double(), dist.double()
    else:
        wlo, whi = (1 - dist).double(), dist.double()
    idx = torch.stack([a["lo"], a["hi"]], -1).flatten(-2)
    w = torch.stack([wlo * ok, whi * ok], -1).flatten(-2)
    d = torch.stack([-ok, ok], -1).flatten(-2)
    return idx, w, d


def _roi_chunks(N, per_roi):
    step = max(1, CHUNK // max(1, per_roi))
    return [(s, min(N, s + step)) for s in range(0, N, step)]


def _channel_of(output_dim, group_size, P, dev):
    """channel read by (ctop, ph, pw): (ctop * G + gh) * G + gw, gh / gw as deform_geom (float32 products)"""
    G = torch.tensor(float(group_size), dtype=F32, device=dev)
    Pf = torch.tensor(float(P), dtype=F32, device=dev)
    gi = torch.floor((torch.arange(P, device=dev).to(F32) * G) / Pf).long().clamp(0, group_size - 1)
    ctop = torch.arange(output_dim, device=dev).view(-1, 1, 1)
    return (ctop * group_size + gi.view(1, P, 1)) * group_size + gi.view(1, 1, P)


def _ps_terms(data, g, n0, n1, output_dim, group_size, channels_each_class, kind):
    """gathered corner grid of rois n0:n1: (values [n, ctop, P, P, 2S, 2S], wy, wx, dy, dx, flat data index)"""
    B, C, H, W = data.shape
    P = g["P"]
    dev = data.device
    cls = torch.arange(output_dim, device=dev) // channels_each_class
    yi, wy, dy = _axis_tab({k: v[n0:n1] for k, v in g["y"].items()}, kind)     # [n, ncls, P, P(pw), 2S]
    xi, wx, dx = _axis_tab({k: v[n0:n1] for k, v in g["x"].items()}, kind)
    # the rows of a bin depend on ph and, through trans, on pw (likewise the columns): [n, od, P, P, 2S(a), 2S(b)]
    yi, wy, dy = yi[:, cls, ..., :, None], wy[:, cls, ..., :, None], dy[:, cls, ..., :, None]
    xi, wx, dx = xi[:, cls, ..., None, :], wx[:, cls, ..., None, :], dx[:, cls, ..., None, :]
    ch = _channel_of(output_dim, group_size, P, dev).view(1, output_dim, P, P, 1, 1)
    b = g["b"][n0:n1].view(-1, 1, 1, 1, 1, 1)
    flat = ((b * C + ch) * H + yi) * W + xi
    vals = data.reshape(-1)[flat]
    return vals, wy, wx, dy, dx, flat


def deform_psroi_fwd(data, g, *, output_dim, group_size, kind="exact"):
    """pooled output [N, output_dim, P, P] (float64, NCHW order) and the mean of |w * v| per bin.  data: float64 NCHW."""
    N, P = g["N"], g["P"]
    ncls = g["ncls"]
    ce = output_dim // ncls
    cnt = ps_count(g).double()
    cls = torch.arange(output_dim, device=data.device) // ce
    out = torch.zeros(N, output_dim, P, P, dtype=F64, device=data.device)
    mag = torch.zeros_like(out)
    for n0, n1 in _roi_chunks(N, output_dim * P * P * (2 * g["S"]) ** 2):
        v, wy, wx, _, _, _ = _ps_terms(data, g, n0, n1, output_dim, group_size, ce, kind)
        t = wy * wx * v
        out[n0:n1] = t.sum((-2, -1))
        mag[n0:n1] = t.abs().sum((-2, -1))
    c = cnt[:, cls]
    inv = torch.where(c > 0, 1.0 / c.clamp(min=1), torch.zeros_like(c))
    return out * inv, mag * inv


def deform_psroi_bwd(top_diff, data, g, *, output_dim, group_size, trans_std, no_trans, kind="exact"):
    """float64 gradients of deform_psroi_fwd: dict(data_diff NCHW, dd_mag, dd_terms, trans_diff [N, 2*ncls, part,
    part], td_mag, td_bins).  top_diff: [N, output_dim, P, P] (float32 values, NCHW order).  dd_terms counts the
    (bin, sample, corner) contributions per element; td_bins the bins per trans element."""
    B, C, H, W = data.shape
    N, P, S, ncls, part = g["N"], g["P"], g["S"], g["ncls"], g["part"]
    ce = output_dim // ncls
    dev = data.device
    cnt = ps_count(g).double()
    cls = torch.arange(output_dim, device=dev) // ce
    c = cnt[:, cls]
    diff = torch.where(c > 0, top_diff.double() / c.clamp(min=1), torch.zeros_like(c))     # [N, od, P, P]
    dd = torch.zeros(B * C * H * W, dtype=F64, device=dev)
    ddm, ddt = torch.zeros_like(dd), torch.zeros_like(dd)
    td = torch.zeros(N, ncls, 2, part, part, dtype=F64, device=dev)
    tdm, tdb = torch.zeros_like(td), torch.zeros_like(td)
    pi = g["part_idx"]
    for n0, n1 in _roi_chunks(N, output_dim * P * P * (2 * S) ** 2):
        v, wy, wx, dy, dx, flat = _ps_terms(data, g, n0, n1, output_dim, group_size, ce, kind)
        dv = diff[n0:n1, ..., None, None]
        t = wy * wx * dv
        t, flat_b = torch.broadcast_tensors(t, flat)
        dd.index_add_(0, flat_b.reshape(-1), t.reshape(-1))
        ddm.index_add_(0, flat_b.reshape(-1), t.abs().reshape(-1))
        ddt.index_add_(0, flat_b.reshape(-1), (t != 0).double().reshape(-1))
        if no_trans:
            continue
        n = n1 - n0
        rw = g["roi_w"][n0:n1].double().view(-1, 1, 1, 1)
        rh = g["roi_h"][n0:n1].double().view(-1, 1, 1, 1)
        gx = (wy * dx * v * dv).sum((-2, -1)) * trans_std * rw          # [n, od, P, P]
        gy = (dy * wx * v * dv).sum((-2, -1)) * trans_std * rh
        gxm = (wy * dx.abs() * v.abs() * dv.abs()).sum((-2, -1)) * trans_std * rw
        gym = (dy.abs() * wx * v.abs() * dv.abs()).sum((-2, -1)) * trans_std * rh
        nz = (c[n0:n1] > 0).double()
        tix = ((((torch.arange(n0, n1, device=dev).view(-1, 1, 1, 1) * ncls + cls.view(1, -1, 1, 1)) * 2) * part
                + pi.view(1, 1, P, 1)) * part + pi.view(1, 1, 1, P)).expand(n, output_dim, P, P).reshape(-1)
        for k, (a, am) in enumerate(((gx, gxm), (gy, gym))):
            off = k * part * part
            td.view(-1).index_add_(0, tix + off, a.reshape(-1))
            tdm.view(-1).index_add_(0, tix + off, am.reshape(-1))
            tdb.view(-1).index_add_(0, tix + off, nz.expand(n, output_dim, P, P).reshape(-1))
    return dict(data_diff=dd.view(B, C, H, W), dd_mag=ddm.view(B, C, H, W), dd_terms=ddt.view(B, C, H, W),
                trans_diff=td.view(N, 2 * ncls, part, part), td_mag=tdm.view(N, 2 * ncls, part, part),
                td_bins=tdb.view(N, 2 * ncls, part, part))


def psroi_bins(rois, *, H, W, spatial_scale, pooled):
    """psroi_bin of psroi.cu: int64 [N, P, P] hstart / hend (rows ph) and wstart / wend (columns pw), batch index"""
    dev = rois.device
    P = pooled
    f = lambda v: torch.tensor(v, dtype=F32, device=dev)
    sc = f(spatial_scale)
    r = _round_away(rois[:, 1:5])
    sw, sh = r[:, 0] * sc, r[:, 1] * sc
    ew = (r[:, 2].double() + 1.0).to(F32) * sc
    eh = (r[:, 3].double() + 1.0).to(F32) * sc
    rw = torch.clamp((ew - sw).double(), min=0.1).to(F32)
    rh = torch.clamp((eh - sh).double(), min=0.1).to(F32)
    bw, bh = rw / f(P), rh / f(P)
    p = torch.arange(P, device=dev).to(F32)
    hs = torch.floor(p.view(1, P) * bh.view(-1, 1) + sh.view(-1, 1)).long().clamp(0, H)
    he = torch.ceil((p + 1).view(1, P) * bh.view(-1, 1) + sh.view(-1, 1)).long().clamp(0, H)
    ws = torch.floor(p.view(1, P) * bw.view(-1, 1) + sw.view(-1, 1)).long().clamp(0, W)
    we = torch.ceil((p + 1).view(1, P) * bw.view(-1, 1) + sw.view(-1, 1)).long().clamp(0, W)
    N = rois.shape[0]
    return dict(b=rois[:, 0].long(), hs=hs.view(N, P, 1).expand(N, P, P), he=he.view(N, P, 1).expand(N, P, P),
                ws=ws.view(N, 1, P).expand(N, P, P), we=we.view(N, 1, P).expand(N, P, P))


def psroi_bins_array(bins, output_dim):
    """oracle_psroi_fwd's bins [N*output_dim*P*P, 4] = hstart, hend, wstart, wend (NCHW order)"""
    N, P, _ = bins["hs"].shape
    t = torch.stack([bins["hs"], bins["he"], bins["ws"], bins["we"]], -1)
    return t[:, None].expand(N, output_dim, P, P, 4).reshape(-1, 4).int()


def psroi_fwd(data, bins, *, output_dim, group_size):
    """box means [N, output_dim, P, P] (float64) and the mean of |data| over the box, from float64 integral images"""
    B, C, H, W = data.shape
    N, P, _ = bins["hs"].shape
    I = torch.zeros(B, C, H + 1, W + 1, dtype=F64, device=data.device)
    Ia = torch.zeros_like(I)
    I[:, :, 1:, 1:] = data.double().cumsum(2).cumsum(3)
    Ia[:, :, 1:, 1:] = data.double().abs().cumsum(2).cumsum(3)
    ch = _channel_of(output_dim, group_size, P, data.device).view(1, output_dim, P, P)
    b = bins["b"].view(N, 1, 1, 1)
    hs, he, ws, we = (bins[k].reshape(N, 1, P, P) for k in ("hs", "he", "ws", "we"))

    def box(T):
        return T[b, ch, he, we] - T[b, ch, hs, we] - T[b, ch, he, ws] + T[b, ch, hs, ws]
    area = ((he - hs) * (we - ws)).double()
    empty = (he <= hs) | (we <= ws)
    a = torch.where(empty, torch.ones_like(area), area)
    out = torch.where(empty, torch.zeros_like(area), box(I) / a)
    mag = torch.where(empty, torch.zeros_like(area), box(Ia) / a)
    return out, mag


def psroi_bwd(top_diff, bins, data_shape, *, output_dim, group_size):
    """float64 data_diff (NCHW) of psroi_fwd, its |terms| sum and the number of bins adding to each element, through a
    2-D difference array and two cumulative sums"""
    B, C, H, W = data_shape
    N, P, _ = bins["hs"].shape
    dev = top_diff.device
    ch = _channel_of(output_dim, group_size, P, dev).view(1, output_dim, P, P)
    b = bins["b"].view(N, 1, 1, 1)
    hs, he, ws, we = (bins[k].reshape(N, 1, P, P) for k in ("hs", "he", "ws", "we"))
    empty = (he <= hs) | (we <= ws)
    area = ((he - hs) * (we - ws)).double().clamp(min=1)
    v = torch.where(empty, torch.zeros_like(area), top_diff.double() / area)
    one = (~empty).double().expand_as(v)
    outs = []
    for val in (v, v.abs(), one):
        D = torch.zeros(B, C, H + 1, W + 1, dtype=F64, device=dev)
        for (yy, xx, s) in ((hs, ws, 1), (hs, we, -1), (he, ws, -1), (he, we, 1)):
            idx = (((b * C + ch) * (H + 1) + yy) * (W + 1) + xx).expand_as(val)
            D.view(-1).index_add_(0, idx.reshape(-1), (s * val).reshape(-1))
        outs.append(D.cumsum(2).cumsum(3)[:, :, :H, :W])
    # prefix sums leave ~1e-16 * (sum over the plane) where no bin adds anything: those elements are exactly 0
    terms = outs[2].round()
    covered = terms > 0
    return outs[0] * covered, outs[1] * covered, terms


def edge_rois(H, W, B, pooled, sample_per_part, n_random, gen, stride=16):
    """float32 rois [n, 5] in image coordinates (feature stride `stride`) on an H x W map of B images: n_random inside,
    then one of each edge case -- crossing each border, fully outside on either side (no sample: count 0), degenerate
    (end before start: the 0.1 minimum extent), x.5 corners (roundf ties away from zero), first samples exactly on
    -0.5 and last samples exactly on extent - 0.5, all on the last image of the batch."""
    P, S = pooled, sample_per_part
    xs = torch.rand(n_random, 2, generator=gen) * (W * stride) - 0.25 * stride
    ys = torch.rand(n_random, 2, generator=gen) * (H * stride) - 0.25 * stride
    r = torch.stack([torch.randint(0, B, (n_random,), generator=gen).float(), xs.min(1).values, ys.min(1).values,
                     xs.max(1).values, ys.max(1).values], 1)
    Wc, Hc = W * stride, H * stride
    k = P * S                  # a roi of k feature pixels from an integer pixel puts its samples on whole pixels - 0.5
    edge = [
        (-40, 8, 100, 40), (Wc - 100, 8, Wc + 60, 40), (8, -40, 40, 100), (8, Hc - 100, 40, Hc + 60),   # borders
        (-60, -60, Wc + 60, Hc + 60),                                                                   # all of it
        (Wc + 100, 0, Wc + 300, 50), (-400, 0, -200, 50), (0, Hc + 64, 50, Hc + 300), (0, -500, 50, -300),  # outside
        (50, 50, 20, 20), (5, 5, 5, 5), (30, 30, 30.4, 70),                                            # degenerate
        (10.5, 24.5, 31.5, 40.5), (-0.5, 2.5, 17.5, 33.5), (-1.5, -0.5, 0.5, 1.5),                      # x.5 ties
        (0, 0, k * stride - 1, k * stride - 1),                                                         # first on -0.5
        (stride * (W - k + 1), stride * (H - k + 1), stride * (W + 1) - 1, stride * (H + 1) - 1),       # last on W-0.5
    ]
    e = torch.tensor([[B - 1] + list(map(float, c)) for c in edge], dtype=F32)
    return torch.cat([r, e]).contiguous()
