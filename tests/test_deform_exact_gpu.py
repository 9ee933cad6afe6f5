"""Deformable convolution (csrc/deform_conv.cu) and (Deformable)PSROIPooling (csrc/psroi.cu) against the float64
references of tests/deform_ref.py, on every launch path.

Each case has its own seeded generator and an id naming its shape.  The references evaluate the sample geometry in
float32 in the kernels' order (pinned bit for bit against the C oracle by tests/test_deform_reference_cpu.py) and
everything after it in float64.  u = 2^-24 (half an fp32 ulp); mag = the float64 sum of |terms| the result is made of;
n = the number of terms an element receives (the length of its chain of atomic additions); P = the prefilled value an
output accumulates onto.  Bounds are worst-case operation counts, not fitted tolerances:

Deformable convolution
- col: bit-equal to a gather of x for zero / whole-pixel offsets (fp32 and bf16); otherwise 4u * mag against the kernel's
  fp32 weights (four products, three additions), plus half a bf16 ulp of the result for bf16 storage.
- dx, fp64-scratch entry: the products are exact in fp64 and summed in fp64; the result is rounded to fp32 and added to
  P in fp32: u (|S| + |P + S|) + n 2^-53 mag.
- dx, float-atomic entry (sniper_deform_col2im): (n + 2) u (mag + |P|).
- doffset: (16 + cpg / 128) u mag (+ u |Q + S| onto the prefill Q when cpg > 128): the 1 - l rounding, the 4-channel
  lane sum, the 32-lane shuffle tree and the cpg / 128 atomics.  Written (NaN prefill survives nowhere) at cpg = 128,
  accumulated otherwise; columns >= 2 dg KH KW of a padded offset row stay untouched.
PSROI
- counts and sample indices: exact everywhere; the oracle-order forward (SNIPER_PSROI_EXACT=1) is byte-equal to the
  generic kernel, which is byte-equal to the C oracle; both within (S^2 + 8) u * mag of float64.
- separable forward: ((2S)^2 + 4S + 4) u * mag (summed axis weights, at most (2S)^2 fma terms, one reciprocal).
- data gradient: generic (n + 6) u (mag + |P|); separable, float atomics (2S + 4 + n) u (mag + |P|); fp64 scratch
  (2S + 3) u mag + u (|S| + |P + S|).
- trans gradient: generic (S^2 + 17 + b) u mag; separable ((2S)^2 CC + 4S + 20 + b) u mag, with b the bins adding to
  the element and CC = C / 128.  The separable bound charges every lane the worst-case (2S)^2 CC sequential
  additions; the measured error stays below 1e-2 of it because a bin touches only ~3 x 3 distinct pixels and the
  partial sums do not grow monotonically.  The bound is kept worst-case rather than fitted.
- PSROIPooling: forward (area + 1) u mag, backward (n + 1) u mag (+ 1e-12 max mag for the reference's prefix sums).
Reproducibility of the fp64-scratch entry points (deformable dx, PSROI data and trans gradients).  Their fp64 sums of
exact products still round, so the order in which the atomics arrive can move a sum's last fp64 bits, and an fp32
result whose sum lies that close to a rounding boundary.  Two runs are therefore checked for the mechanism, not for
byte-identity: each result is bit for bit prefill + (float) fp64 sum, the two runs' sums differ by at most
(n + 1) 2^-52 mag, and an element may differ between the runs only where its two sums round to different floats; every
such element is listed by the report.  The single-writer doffset (cpg = 128) is byte-identical across runs.

Every case draws its data from a generator seeded with the crc32 of its key, so a failing id reproduces.
`test_zz_report` prints the worst error / bound per class (run with -s).  Measured on an H100 80GB HBM3 (700 W), two
runs: col 0.89 fp32 / 0.99 bf16; dx 1.00 (fp64 scratch) / 0.58 (float atomics); doffset 0.05 written / 0.03
accumulated (the bound charges the lane-sum and shuffle roundings at their worst; they cancel); PSROI forward 0.48
generic / 0.34 separable; data gradient 0.99 fp64 scratch / 0.47 generic / 0.30 separable; trans gradient 0.57 generic /
0.008 separable (see above); PSROIPooling 0.56 forward / 0.52 backward; run-to-run fp64 sums within 0.31 of their bound,
no element moved in either run.  Whole file: 157 tests in 18 s."""
import zlib

import numpy as np
import pytest

import deform_ref as R
import oracle_lib as O

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24
WORST = {}


def _note(what, err, bound):
    import torch
    ratio = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, float("inf"), 0.0).double())
    i = int(ratio.reshape(-1).argmax())
    r = (float(ratio.reshape(-1)[i]), float(err.reshape(-1)[i]), float(bound.reshape(-1)[i]))
    if what not in WORST or r[0] > WORST[what][0]:
        WORST[what] = r


def _within(what, got, ref, bound):
    import torch
    got = got.double()
    assert bool(torch.isfinite(got).all()), what + ": NaN / Inf in the result"
    err = (got - ref).abs()
    bound = torch.broadcast_to(bound, err.shape)
    _note(what, err, bound)
    bad = err > bound
    assert not bool(bad.any()), "%s: %d elements out of bound, worst excess %.3e" % (
        what, int(bad.sum()), float((err - bound).max()))


def _seed(*key):
    """a seed that depends on the case only (str hashes are salted per process)"""
    return zlib.crc32(repr(key).encode())


def _gen(*key):
    import torch
    g = torch.Generator(device=DEV)
    g.manual_seed(_seed(*key))
    return g


MOVED = []                   # (what, flat index, run 1, run 2, fp64 sum 1, fp64 sum 2) of every element two runs disagree on


def _fp64_scratch_repro(what, run, P, n_terms, mag):
    """Two runs of an fp64-scratch entry point.  `run()` returns (fp32 result, the fp64 sums it was made from).  The
    fp64 sums of exact products still round, so arrival order may move a sum's last fp64 bits -- by at most
    (n + 1) 2^-52 mag -- and, where a sum lies that close to an fp32 rounding boundary, the fp32 result.  Checked: each
    result is bit for bit P + (float)sum, the two sums differ within that bound, and every element that moved between
    the runs is one whose two sums round to different floats.  Each moved element is recorded for the report."""
    import torch
    (o1, a1), (o2, a2) = run(), run()
    for o, a in ((o1, a1), (o2, a2)):
        assert torch.equal(o, P + a.float()), what + ": result is not prefill + (float) fp64 sum"
    _within(what + " run-to-run fp64 sums", a2, a1, (n_terms + 1) * 2.0 ** -52 * mag * 1.01 + 2.0 ** -1074)
    moved = o1 != o2
    assert not bool((moved & (a1.float() == a2.float())).any()), what + ": moved without a different fp64 sum"
    for i in moved.reshape(-1).nonzero().reshape(-1)[:16].tolist():
        MOVED.append((what, i, float(o1.reshape(-1)[i]), float(o2.reshape(-1)[i]), float(a1.reshape(-1)[i]),
                      float(a2.reshape(-1)[i])))


# ---------------------------------------------------------------------------------------------- deformable conv
# (dtype, NB, H, W, C, dgroups, KH, KW, stride, dil, pad, off_ld or 0 = exact)
DC_GRID = []
for _dt in ("float32", "bfloat16"):
    DC_GRID += [(_dt, 2, 10, 13, 128, 1, 3, 3, 1, 1, 1, 0), (_dt, 2, 9, 7, 256, 1, 3, 3, 2, 2, 2, 96),
                (_dt, 1, 6, 11, 512, 1, 5, 5, 1, 2, 2, 0), (_dt, 2, 1, 17, 256, 2, 1, 3, 1, 1, 0, 0),
                (_dt, 2, 13, 1, 1024, 2, 3, 3, 2, 1, 1, 96), (_dt, 1, 2, 3, 128, 1, 5, 5, 1, 2, 4, 0),
                (_dt, 2, 10, 16, 512, 4, 3, 3, 1, 2, 2, 96), (_dt, 1, 7, 9, 1024, 8, 1, 3, 2, 2, 1, 0),
                (_dt, 2, 5, 6, 256, 2, 1, 1, 1, 1, 0, 0)]
DC_BIG = [(_dt, 20, 32, 32, 512, 4, 3, 3, 1, 2, 2, 96) for _dt in ("float32", "bfloat16")] + \
         [("bfloat16", 2, 50, 80, 512, 4, 3, 3, 1, 2, 2, 96)]
OFFSETS = ["sigma0.05", "sigma1.5", "edges", "integer", "zero", "far"]


def _dc_id(c):
    return "%s-%dx%dx%dx%d-dg%d-k%dx%d-s%d-d%d-p%d-ld%d" % ((("fp32" if c[0] == "float32" else "bf16"),) + c[1:])


def _offsets(kind, g, NB, H, W, KH, KW, stride, dil, pad, dg, off_ld):
    """float32 [NB, Ho, Wo, off_ld]; the columns past 2 dg KH KW hold a sentinel"""
    import torch
    Ho, Wo = R.out_extent(H, KH, stride, dil, pad), R.out_extent(W, KW, stride, dil, pad)
    K2 = dg * 2 * KH * KW
    shape = (NB, Ho, Wo, dg, KH * KW, 2)
    if kind.startswith("sigma"):
        o = torch.randn(shape, generator=g, device=DEV) * float(kind[5:])
    elif kind == "integer":
        o = torch.randint(-3, 4, shape, generator=g, device=DEV).float()
    elif kind == "zero":
        o = torch.zeros(shape, device=DEV)
    elif kind == "far":
        o = torch.randint(0, 2, shape, generator=g, device=DEV).float() * 4 * max(H, W) - 2 * max(H, W)
    else:
        # per tap, aim h_im / w_im at -1, -2^-20, 0, 0.5, just below X - 1, X - 1, X - 0.5, just below X and X
        # ("just below" = the next float32 down: X - 2^-20 is not representable once X >= 16); targets cycle over the
        # samples.  o = fl(target - base) lands exactly wherever that difference is exact in float32, which
        # _edge_hits() confirms for every target
        th, tw = _edge_targets(H), _edge_targets(W)
        base_h, base_w = _edge_bases(Ho, Wo, KH, KW, stride, dil, pad)
        k = torch.arange(NB * Ho * Wo * dg * KH * KW, device=DEV).view(shape[:-1])
        o = torch.stack([th[k % 9] - base_h.float(), tw[(k // 9 + k) % 9] - base_w.float()], -1)
    out = torch.full((NB, Ho, Wo, off_ld or K2), 7.0, device=DEV)
    out[..., :K2] = o.reshape(NB, Ho, Wo, K2)
    return out


def _edge_targets(X):
    import torch
    below = lambda v: float(np.nextafter(np.float32(v), np.float32(-np.inf)))
    return torch.tensor([-1, -2.0 ** -20, 0, 0.5, below(X - 1), X - 1, X - 0.5, below(X), X], device=DEV)


def _edge_bases(Ho, Wo, KH, KW, stride, dil, pad):
    import torch
    tap = torch.arange(KH * KW, device=DEV)
    base_h = (torch.arange(Ho, device=DEV) * stride - pad).view(1, Ho, 1, 1, 1) + ((tap // KW) * dil).view(1, 1, 1, 1, -1)
    base_w = (torch.arange(Wo, device=DEV) * stride - pad).view(1, 1, Wo, 1, 1) + ((tap % KW) * dil).view(1, 1, 1, 1, -1)
    return base_h, base_w


def _edge_hits(off, H, W, KH, KW, stride, dil, pad, dg):
    """which of the nine targets some sample's h_im (w_im) equals exactly, computed as the kernel does"""
    import torch
    NB, Ho, Wo, _ = off.shape
    o = off[..., :dg * 2 * KH * KW].reshape(NB, Ho, Wo, dg, KH * KW, 2)
    base_h, base_w = _edge_bases(Ho, Wo, KH, KW, stride, dil, pad)
    h_im, w_im = base_h.float() + o[..., 0], base_w.float() + o[..., 1]
    return ([bool((h_im == t).any()) for t in _edge_targets(H)], [bool((w_im == t).any()) for t in _edge_targets(W)])


def _dc_case(case, kind, salt=""):
    import torch
    dt, NB, H, W, C, dg, KH, KW, st, dil, pad, ld = case
    g = _gen(case, kind, salt)
    x = torch.randn(NB, H, W, C, generator=g, device=DEV).to(getattr(torch, dt))
    off = _offsets(kind, g, NB, H, W, KH, KW, st, dil, pad, dg, ld)
    return g, x, off, dict(kh=KH, kw=KW, stride=st, dil=dil, pad=pad, dgroups=dg)


def _col_bound(ref_mag, ref, dt):
    import torch
    b = 4 * U * ref_mag + 4 * 2.0 ** -149
    if dt != torch.float32:
        b = b + (ref.abs() + b) * 2.0 ** -8 * 1.01
    return b


def _dc_forward_checks(case, kind, x, off, kw):
    import torch
    from sniper_b200 import ops
    NB, H, W, C = x.shape
    Ho, Wo = off.shape[1], off.shape[2]
    out = torch.full((NB * Ho * Wo, kw["kh"] * kw["kw"] * C), float("nan"), device=DEV, dtype=x.dtype)
    col = ops.deform_im2col(x, off, out=out, **kw)
    ref, mag = R.dc_im2col(x, off, kw["kh"], kw["kw"], kw["stride"], kw["dil"], kw["pad"], kw["dgroups"], kind="kernel")
    if kind in ("integer", "zero", "far"):
        # whole-pixel samples: col is a shifted copy of x (zeros outside), bit for bit
        assert bool(torch.isfinite(col.float()).all())
        assert torch.equal(col, ref.to(x.dtype)), "col is not a bit-exact gather of x"
        _note("col whole-pixel (bit-equal)", torch.zeros(1, dtype=torch.float64), torch.ones(1, dtype=torch.float64))
    _within("col " + ("fp32" if x.dtype == torch.float32 else "bf16"), col, ref, _col_bound(mag, ref, x.dtype))
    return col


def _dc_backward_checks(case, kind, g, x, off, kw, reps=True):
    import torch
    from sniper_b200 import ops
    NB, H, W, C = x.shape
    KK = kw["kh"] * kw["kw"]
    dg = kw["dgroups"]
    cpg = C // dg
    K2 = dg * 2 * KK
    Ho, Wo = off.shape[1], off.shape[2]
    dcol = torch.randn(NB * Ho * Wo, KK * C, generator=g, device=DEV).to(x.dtype)
    G = R.dc_col2im(dcol, x, off, kw["kh"], kw["kw"], kw["stride"], kw["dil"], kw["pad"], dg, kind="kernel")
    P = torch.randn(NB, H, W, C, generator=g, device=DEV)
    Q = torch.randn(off.shape, generator=g, device=DEV)
    if cpg == 128:
        Q[..., :K2] = float("nan")          # written, not accumulated: the NaN must not survive
    runs = []
    for _ in range(2 if reps else 1):
        dx, doff = ops.deform_col2im(dcol, x, off, dx=P.clone(), doffset=Q.clone(), **kw)
        runs.append((dx, doff))
    dx, doff = runs[0]
    S = G["dx"]
    b = U * (S.abs() + (P.double() + S).abs()) + G["dx_terms"] * 2.0 ** -53 * G["dx_mag"] + 2.0 ** -149
    _within("dx fp64 scratch", dx, P.double() + S, b)
    pre = 0.0 if cpg == 128 else Q[..., :K2].double()
    ref = pre + G["doff"]
    bd = (16 + cpg // 128) * U * G["doff_mag"] + U * ref.abs() + 2.0 ** -149
    _within("doffset " + ("written (cpg 128)" if cpg == 128 else "accumulated (cpg > 128)"), doff[..., :K2], ref, bd)
    assert torch.equal(doff[..., K2:], Q[..., K2:]), "padding columns of doffset were written"
    from sniper_b200 import _lib
    from sniper_b200.ops import _ptr, _sdt, _stream
    if reps:
        if cpg == 128:      # one warp writes each element: the same bits every run
            assert doff.cpu().numpy().tobytes() == runs[1][1].cpu().numpy().tobytes(), "doffset differs between runs"

        def run():
            acc = torch.zeros(x.shape, dtype=torch.float64, device=DEV)
            dx_, doff_ = P.clone(), Q.clone()
            rc = _lib.lib().sniper_deform_col2im_fp64acc(_ptr(dcol), _ptr(x), _ptr(off), NB, H, W, C, kw["kh"], kw["kw"],
                                                         kw["stride"], kw["dil"], kw["pad"], dg, off.stride(2), _ptr(dx_),
                                                         _ptr(doff_), _sdt(x), _ptr(acc), acc.numel(), _stream())
            assert rc == 0, _lib.lib().sniper_last_error().decode()
            return dx_, acc
        _fp64_scratch_repro("dx fp64 scratch", run, P, G["dx_terms"], G["dx_mag"])
    # the float-atomic entry point
    dx2, doff2 = P.clone(), Q.clone()
    rc = _lib.lib().sniper_deform_col2im(_ptr(dcol), _ptr(x), _ptr(off), NB, H, W, C, kw["kh"], kw["kw"], kw["stride"],
                                         kw["dil"], kw["pad"], dg, off.stride(2), _ptr(dx2), _ptr(doff2), _sdt(x),
                                         _stream())
    assert rc == 0, _lib.lib().sniper_last_error().decode()
    b2 = (G["dx_terms"] + 2) * U * (G["dx_mag"] + P.double().abs()) * 1.01 + 2.0 ** -149
    _within("dx float atomics", dx2, P.double() + S, b2)
    _within("doffset float atomics", doff2[..., :K2], ref, bd)


@pytest.mark.parametrize("kind", OFFSETS)
@pytest.mark.parametrize("case", DC_GRID, ids=_dc_id)
def test_deform_conv(case, kind):
    g, x, off, kw = _dc_case(case, kind)
    if kind == "edges":
        hh, ww = _edge_hits(off, x.shape[1], x.shape[2], kw["kh"], kw["kw"], kw["stride"], kw["dil"], kw["pad"],
                            kw["dgroups"])
        assert all(hh) and all(ww), ("edge targets not reached exactly", hh, ww)
    _dc_forward_checks(case, kind, x, off, kw)
    _dc_backward_checks(case, kind, g, x, off, kw, reps=kind in ("sigma1.5", "edges"))


@pytest.mark.parametrize("case", DC_BIG, ids=_dc_id)
def test_deform_conv_product_shapes(case):
    """training (20 chips x 32 x 32 x 512, offsets like the offset conv's fp32 output) and inference (2 x 50 x 80)"""
    g, x, off, kw = _dc_case(case, "sigma1.5")
    _dc_forward_checks(case, "sigma1.5", x, off, kw)
    _dc_backward_checks(case, "sigma1.5", g, x, off, kw, reps=True)


# ---------------------------------------------------------------------------------------------- PSROI
# (layout, C (= output_dim * G^2), G, ncls, pooled, part, S, B, H, W)
PS_GRID = []
for _C in (128, 256, 512):
    for _S in (1, 2, 3, 4):
        PS_GRID.append((1, _C, 1, 1, 7, 7, _S, 2, 12, 20))
PS_GRID += [(1, 256, 1, 1, 7, 3, 4, 3, 1, 30), (1, 128, 1, 1, 3, 3, 4, 2, 9, 5),            # part != pooled, height 1
            (1, 256, 1, 1, 7, 7, 5, 2, 12, 20), (1, 18, 3, 1, 3, 3, 4, 2, 14, 14),          # generic: S = 5, G = 3
            (1, 256, 1, 2, 7, 7, 4, 2, 12, 20), (0, 256, 1, 1, 7, 7, 4, 2, 20, 12),         # two classes, NCHW
            (0, 18, 3, 2, 3, 3, 2, 2, 1, 30)]


def _ps_id(c):
    return "%s-C%d-g%d-cls%d-P%d-part%d-S%d-B%d-%dx%d" % ((("nchw", "nhwc")[c[0]],) + tuple(c[1:]))


def _ps_inputs(case, n_random=40, salt=""):
    import torch
    lay, C, G, ncls, P, part, S, B, H, W = case
    g = _gen(case, salt)
    data = torch.randn(B, C, H, W, generator=g, device=DEV)
    gc = torch.Generator()
    gc.manual_seed(_seed(case, salt))
    rois = R.edge_rois(H, W, B, P, S, n_random, gc).to(DEV)
    N = rois.shape[0]
    trans = torch.randn(N, 2 * ncls, part, part, generator=g, device=DEV) * 1.5
    return data, rois, trans


def _nchw(t, lay):
    return t if lay == 0 else t.permute(0, 3, 1, 2)


def _stored(t, lay):
    return (t if lay == 0 else t.permute(0, 2, 3, 1)).contiguous()


def _misaligned(t):
    """a copy of t whose storage starts one float past a 16-byte boundary"""
    import torch
    buf = torch.empty(t.numel() + 4, device=t.device, dtype=t.dtype)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def _ps_fwd_checks(case, no_trans, monkeypatch):
    import torch
    from sniper_b200 import ops
    lay, C, G, ncls, P, part, S, B, H, W = case
    if no_trans:
        ncls = 1
    od = C // (G * G)
    data, rois, trans = _ps_inputs(case, salt=no_trans)
    if no_trans:
        trans = trans[:, :2]
    kw = dict(spatial_scale=0.0625, output_dim=od, group_size=G, pooled_size=P, part_size=part, sample_per_part=S,
              trans_std=0.1, no_trans=no_trans)
    d = _stored(data, lay)
    geo = R.ps_geom(rois, None if no_trans else trans, H=H, W=W, spatial_scale=0.0625, pooled=P, part_size=part,
                    sample_per_part=S, trans_std=0.1, no_trans=no_trans, ncls=ncls)
    ce = od // ncls
    cnt_ref = R.ps_count(geo)[:, torch.arange(od, device=DEV) // ce].float()
    ref, mag = R.deform_psroi_fwd(data.double(), geo, output_dim=od, group_size=G)
    # generic kernel (sample indices requested): indices and counts exact, within the per-sample bound
    out_g, cnt_g, sidx = ops.deform_psroi_fwd(d, rois, trans, layout=lay, want_sample_idx=True, **kw)
    assert torch.equal(sidx, R.ps_sample_idx(geo, W, od, ce))
    assert torch.equal(_nchw(cnt_g, lay), cnt_ref)
    _within("psroi fwd generic", _nchw(out_g, lay), ref, (S * S + 8) * U * mag + 2.0 ** -149)
    # the generic kernel is the C oracle (the reference's float32 operation order) bit for bit
    o_out, o_cnt, o_sidx = O.deform_psroi_fwd(data.cpu().numpy(), rois.cpu().numpy(), trans.cpu().numpy(),
                                              spatial_scale=0.0625, output_dim=od, group_size=G, pooled=P,
                                              part_size=part, spp=S, trans_std=0.1, no_trans=no_trans)
    assert _nchw(out_g, lay).contiguous().cpu().numpy().tobytes() == o_out.tobytes(), "generic forward is not the oracle"
    assert np.array_equal(_nchw(cnt_g, lay).cpu().numpy(), o_cnt)
    assert np.array_equal(sidx.cpu().numpy(), o_sidx)
    assert bool((_nchw(out_g, lay)[cnt_ref == 0] == 0).all())
    fast = lay == 1 and G == 1 and ncls == 1 and S <= 4 and C in (128, 256, 512)
    # oracle order on the warp-per-bin kernel: the same bits as the generic kernel
    monkeypatch.setenv("SNIPER_PSROI_EXACT", "1")
    out_e, cnt_e, _ = ops.deform_psroi_fwd(d, rois, trans, layout=lay, **kw)
    monkeypatch.delenv("SNIPER_PSROI_EXACT")
    assert torch.equal(cnt_e, cnt_g)
    assert out_e.cpu().numpy().tobytes() == out_g.cpu().numpy().tobytes(), "oracle-order forward differs in bits"
    out_s, cnt_s, _ = ops.deform_psroi_fwd(d, rois, trans, layout=lay, **kw)
    assert torch.equal(cnt_s, cnt_g)
    k = ((2 * S) ** 2 + 4 * S + 4) if fast else (S * S + 8)
    _within("psroi fwd separable" if fast else "psroi fwd generic", _nchw(out_s, lay), ref, k * U * mag + 2.0 ** -149)
    if fast:
        # misaligned data or outputs take the generic kernel: the generic kernel's bits
        from sniper_b200 import _lib
        from sniper_b200.ops import _ptr, _stream
        o_m = _misaligned(torch.zeros_like(out_g))
        c_m = _misaligned(torch.zeros_like(out_g))
        for dd_, oo, cc in ((_misaligned(d), torch.empty_like(out_g), None), (d, o_m, None), (d, torch.empty_like(out_g), c_m)):
            rc = _lib.lib().sniper_deform_psroi_fwd(_ptr(dd_), _ptr(rois), _ptr(None if no_trans else trans), rois.shape[0],
                                                    C, H, W, 0.0625, od, G, P, part, S, 0.1, int(no_trans), ncls, lay,
                                                    _ptr(oo), _ptr(cc), None, _stream())
            assert rc == 0, _lib.lib().sniper_last_error().decode()
            assert oo.cpu().numpy().tobytes() == out_g.cpu().numpy().tobytes(), "fallback is not the generic kernel"
            if cc is not None:
                assert torch.equal(cc, cnt_g)
    return data, rois, trans, geo, kw, d


def _ps_bwd_checks(case, no_trans, data, rois, trans, geo, kw, d):
    import torch
    from sniper_b200 import _lib, ops
    from sniper_b200.ops import _ptr, _stream
    lay, C, G, ncls, P, part, S, B, H, W = case
    if no_trans:
        ncls = 1
    od = kw["output_dim"]
    N = rois.shape[0]
    g = _gen(case, no_trans, "bwd")
    td = torch.randn(N, od, P, P, generator=g, device=DEV)
    tdg = _stored(td, lay)
    ref = R.deform_psroi_bwd(td, data.double(), geo, output_dim=od, group_size=G, trans_std=0.1, no_trans=no_trans)
    Pf = torch.randn(d.shape, generator=g, device=DEV)
    Pt = torch.randn(trans.shape, generator=g, device=DEV)
    S_ = ref["data_diff"]
    Pn = _nchw(Pf, lay).double()
    fast = lay == 1 and G == 1 and ncls == 1 and S <= 4 and C in (128, 256, 512)
    CC = C // 128
    kt_sep = ((2 * S) ** 2 * max(CC, 1) + 4 * S + 20 + ref["td_bins"]) * U * ref["td_mag"] + 2.0 ** -149
    kt_gen = (S * S + 17 + ref["td_bins"]) * U * ref["td_mag"] + 2.0 ** -149
    tref = Pt.double() + ref["trans_diff"]
    # ops: the fp64 scratch where the shape qualifies, the generic float-atomic kernel otherwise
    runs = [ops.deform_psroi_bwd(tdg, d, rois, trans, layout=lay, data_diff=Pf.clone(),
                                 trans_diff=None if no_trans else Pt.clone(), **kw) for _ in range(2)]
    dd, tdd = runs[0]
    if fast:
        b = (2 * S + 3) * U * ref["dd_mag"] + U * (S_.abs() + (Pn + S_).abs()) + 2.0 ** -149
        _within("psroi data_diff fp64 scratch", _nchw(dd, lay), Pn + S_, b)
        _within("psroi data_diff fp64 scratch", _nchw(runs[1][0], lay), Pn + S_, b)
        n_data = d.numel()
        n_acc = n_data + (0 if no_trans else trans.numel())

        def run(part_):
            acc = torch.zeros(n_acc, dtype=torch.float64, device=DEV)
            dd_, td_ = Pf.clone(), None if no_trans else Pt.clone()
            rc = _lib.lib().sniper_deform_psroi_bwd_fp64acc(_ptr(tdg), _ptr(d), _ptr(rois), _ptr(None if no_trans else trans),
                                                            N, B, C, H, W, 0.0625, od, G, P, kw["part_size"], S, 0.1,
                                                            int(no_trans), ncls, _ptr(dd_), _ptr(td_), _ptr(acc), n_acc,
                                                            _stream())
            assert rc == 0, _lib.lib().sniper_last_error().decode()
            if part_ == "data":
                return dd_, acc[:n_data].view(d.shape)
            return td_, acc[n_data:].view(trans.shape)
        nhwc = lambda t: t.permute(0, 2, 3, 1)
        _fp64_scratch_repro("psroi data_diff fp64 scratch", lambda: run("data"), Pf, nhwc(ref["dd_terms"]),
                            nhwc(ref["dd_mag"]))
        if not no_trans:
            _fp64_scratch_repro("psroi trans_diff fp64 scratch", lambda: run("trans"), Pt, ref["td_bins"],
                                ref["td_mag"] * 1.01)
        if not no_trans:
            _within("psroi trans_diff fp64 scratch", tdd, tref, kt_sep + U * tref.abs())
    else:
        b = (ref["dd_terms"] + 6) * U * (ref["dd_mag"] + Pn.abs()) * 1.01 + 2.0 ** -149
        _within("psroi data_diff generic", _nchw(dd, lay), Pn + S_, b)
        if not no_trans:
            _within("psroi trans_diff generic", tdd, tref, kt_gen + U * Pt.double().abs() * 2)
    # the float-atomic entry point on the same shape (the separable warp-per-bin kernel when it qualifies)
    dd2, td2 = Pf.clone(), None if no_trans else Pt.clone()
    rc = _lib.lib().sniper_deform_psroi_bwd(_ptr(tdg), _ptr(d), _ptr(rois), _ptr(None if no_trans else trans), N, C, H,
                                            W, 0.0625, od, G, P, kw["part_size"], S, 0.1, int(no_trans), ncls, lay,
                                            _ptr(dd2), _ptr(td2), _stream())
    assert rc == 0, _lib.lib().sniper_last_error().decode()
    if fast:
        b = (2 * S + 4 + ref["dd_terms"]) * U * (ref["dd_mag"] + Pn.abs()) * 1.01 + 2.0 ** -149
        _within("psroi data_diff separable float atomics", _nchw(dd2, lay), Pn + S_, b)
        if not no_trans:
            _within("psroi trans_diff separable float atomics", td2, tref, kt_sep + 2 * U * Pt.double().abs())
        # _fp64acc refuses what the NHWC kernels cannot take; misaligned buffers fall back to the generic kernel
        acc = torch.zeros(1, dtype=torch.float64, device=DEV)
        rc = _lib.lib().sniper_deform_psroi_bwd_fp64acc(_ptr(tdg), _ptr(_misaligned(d)), _ptr(rois),
                                                        _ptr(None if no_trans else trans), N, B, C, H, W, 0.0625, od, G,
                                                        P, kw["part_size"], S, 0.1, int(no_trans), ncls, _ptr(dd2),
                                                        _ptr(td2), _ptr(acc), 1, _stream())
        assert rc == -2
        for name, (a, b_, c_) in (("data", (_misaligned(d), tdg, Pf.clone())), ("top_diff", (d, _misaligned(tdg), Pf.clone())),
                                  ("data_diff", (d, tdg, _misaligned(Pf)))):
            dd3, td3 = ops.deform_psroi_bwd(b_, a, rois, trans, layout=lay, data_diff=c_,
                                            trans_diff=None if no_trans else Pt.clone(), **kw)
            bg = (ref["dd_terms"] + 6) * U * (ref["dd_mag"] + Pn.abs()) * 1.01 + 2.0 ** -149
            _within("psroi data_diff generic", _nchw(dd3, lay), Pn + S_, bg)
            if not no_trans:
                _within("psroi trans_diff generic", td3, tref, kt_gen + 2 * U * Pt.double().abs())
    else:
        b = (ref["dd_terms"] + 6) * U * (ref["dd_mag"] + Pn.abs()) * 1.01 + 2.0 ** -149
        _within("psroi data_diff generic", _nchw(dd2, lay), Pn + S_, b)
    # nothing reaches an element no bin samples
    untouched = ref["dd_terms"] == 0
    assert torch.equal(_nchw(dd, lay)[untouched], _nchw(Pf, lay)[untouched])


@pytest.mark.parametrize("no_trans", [True, False], ids=["no_trans", "trans"])
@pytest.mark.parametrize("case", PS_GRID, ids=_ps_id)
def test_deform_psroi(case, no_trans, monkeypatch):
    data, rois, trans, geo, kw, d = _ps_fwd_checks(case, no_trans, monkeypatch)
    _ps_bwd_checks(case, no_trans, data, rois, trans, geo, kw, d)


def test_deform_psroi_product_head(monkeypatch):
    """the R-FCN head: 20 chips x 300 rois, 256 channels, 7 x 7 bins, 4 x 4 samples, rectangular 32 x 48 maps"""
    case = (1, 256, 1, 1, 7, 7, 4, 20, 32, 48)
    import torch
    lay, C, G, ncls, P, part, S, B, H, W = case
    from sniper_b200 import ops
    g = _gen("head")
    data = torch.randn(B, C, H, W, generator=g, device=DEV)
    gc = torch.Generator()
    gc.manual_seed(5)
    rois = torch.cat([R.edge_rois(H, W, B, P, S, 300 - 17, gc)] * 20).to(DEV)
    rois[:, 0] = torch.arange(20, device=DEV).repeat_interleave(300).float()
    N = rois.shape[0]
    trans = torch.randn(N, 2, P, P, generator=g, device=DEV) * 0.5
    d = _stored(data, lay)
    kw = dict(spatial_scale=0.0625, output_dim=256, group_size=1, pooled_size=P, part_size=P, sample_per_part=S,
              layout=1)
    for no_trans in (True, False):
        geo = R.ps_geom(rois, None if no_trans else trans, H=H, W=W, spatial_scale=0.0625, pooled=P, part_size=P,
                        sample_per_part=S, trans_std=0.1, no_trans=no_trans, ncls=1)
        ref, mag = R.deform_psroi_fwd(data.double(), geo, output_dim=256, group_size=1)
        out, cnt, _ = ops.deform_psroi_fwd(d, rois, trans, no_trans=no_trans, trans_std=0.1, **kw)
        assert torch.equal(_nchw(cnt, 1), R.ps_count(geo)[:, [0] * 256].float())
        _within("psroi fwd separable", _nchw(out, 1), ref, ((2 * S) ** 2 + 4 * S + 4) * U * mag + 2.0 ** -149)
        td = torch.randn(N, 256, P, P, generator=g, device=DEV)
        G_ = R.deform_psroi_bwd(td, data.double(), geo, output_dim=256, group_size=1, trans_std=0.1, no_trans=no_trans)
        dd, tdd = ops.deform_psroi_bwd(_stored(td, 1), d, rois, trans, no_trans=no_trans, trans_std=0.1, **kw)
        S_ = G_["data_diff"]
        _within("psroi data_diff fp64 scratch", _nchw(dd, 1), S_, (2 * S + 3) * U * G_["dd_mag"] + 2 * U * S_.abs())
        if not no_trans:
            kt = ((2 * S) ** 2 * 2 + 4 * S + 20 + G_["td_bins"]) * U * G_["td_mag"] + U * G_["trans_diff"].abs()
            _within("psroi trans_diff fp64 scratch", tdd, G_["trans_diff"], kt)


@pytest.mark.parametrize("lay", [0, 1], ids=["nchw", "nhwc"])
@pytest.mark.parametrize("case", [(2, 2, 3, 20, 24, 3), (2, 1, 7, 1, 13, 7), (3, 256, 1, 9, 30, 7)],
                         ids=lambda c: "B%d-od%d-g%d-%dx%d-P%d" % c)
def test_psroi(case, lay):
    import torch
    from sniper_b200 import ops
    B, od, G, H, W, P = case
    g = _gen("psroi", case, lay)
    data = torch.randn(B, od * G * G, H, W, generator=g, device=DEV)
    gc = torch.Generator()
    gc.manual_seed(11)
    rois = R.edge_rois(H, W, B, P, 1, 40, gc).to(DEV)
    rb = R.psroi_bins(rois, H=H, W=W, spatial_scale=0.0625, pooled=P)
    out, bins = ops.psroi_fwd(_stored(data, lay), rois, spatial_scale=0.0625, output_dim=od, group_size=G,
                              pooled_size=P, layout=lay, want_bins=True)
    assert torch.equal(bins, R.psroi_bins_array(rb, od))
    ref, mag = R.psroi_fwd(data, rb, output_dim=od, group_size=G)
    area = ((rb["he"] - rb["hs"]) * (rb["we"] - rb["ws"])).clamp(min=1).unsqueeze(1).double()
    _within("psroi (plain) fwd", _nchw(out, lay), ref, (area + 1) * U * mag + 1e-12 * float(mag.max()))
    td = torch.randn(rois.shape[0], od, P, P, generator=g, device=DEV)
    shape = data.shape if lay == 0 else (B, H, W, od * G * G)
    dd = ops.psroi_bwd(_stored(td, lay), rois, shape, spatial_scale=0.0625, output_dim=od, group_size=G, pooled_size=P,
                       layout=lay)
    rdd, rmag, terms = R.psroi_bwd(td, rb, data.shape, output_dim=od, group_size=G)
    _within("psroi (plain) bwd", _nchw(dd, lay), rdd, (terms + 1) * U * rmag * 1.01 + 1e-12 * float(rmag.max()))


def test_zz_report():
    for what in sorted(WORST):
        r, e, b = WORST[what]
        print("%-48s worst err/bound %.3e  (err %.3e, bound %.3e)" % (what, r, e, b))
    print("elements that moved between two runs of an fp64-scratch entry point: %d" % len(MOVED))
    for what, i, o1, o2, a1, a2 in MOVED:
        print("  %s [%d]: %.9g / %.9g from fp64 sums %.17g / %.17g" % (what, i, o1, o2, a1, a2))
