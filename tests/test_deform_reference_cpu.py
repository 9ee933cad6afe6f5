"""The float64 references of tests/deform_ref.py, pinned without a device before any kernel is compared with them.

- PSROI geometry: the sample indices and counts of the deformable pooling and the bins of PSROIPooling equal the C
  oracle's (oracle/psroi.c, the reference's source order in float32) bit for bit, on every edge roi of
  deform_ref.edge_rois, on square, rectangular and one-row maps.
- PSROI values: the oracle's float32 pooled values and its double-accumulated gradients lie within the operation-count
  bounds of tests/test_deform_exact_gpu.py of the float64 references (u = 2^-24):
  forward (S^2 + 8) u * mean|w v|; data gradient 5 u * sum|terms|; trans gradient 10 u * sum|terms|.
- Deformable convolution: at 3x3 / stride 1 the float64 im2col matches oracle/torch_graph.deform_conv2d (the graph
  oracle, absolute coordinates) to 1e-12, with offsets on a 2^-10 grid so that the float32 geometry is exact.
- Gradients: the float64 offset / data / trans gradients match central differences of the float64 forwards at points
  whose samples stay clear of pixel boundaries."""
import os
import sys
import zlib

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))

import deform_ref as R          # noqa: E402
import oracle_lib as O          # noqa: E402

U = 2.0 ** -24


def _gen(*key):
    """one generator per case, seeded from the case alone (str hashes are salted per process)"""
    g = torch.Generator()
    g.manual_seed(zlib.crc32(repr(key).encode()))
    return g


# (B, C/od, group_size, H, W, pooled, part, S, ncls)
PS_CASES = [(2, 2, 3, 14, 14, 3, 3, 4, 1), (2, 4, 1, 12, 20, 7, 7, 4, 1), (3, 4, 1, 1, 30, 7, 3, 2, 2),
            (2, 2, 1, 9, 5, 3, 3, 5, 2), (2, 8, 1, 31, 17, 7, 7, 1, 1), (1, 3, 3, 20, 24, 7, 3, 3, 1)]


def _ps_id(c):
    return "B%d-od%d-g%d-%dx%d-P%d-part%d-S%d-cls%d" % c


@pytest.mark.parametrize("no_trans", [True, False], ids=["no_trans", "trans"])
@pytest.mark.parametrize("case", PS_CASES, ids=_ps_id)
def test_deform_psroi_reference_against_oracle(case, no_trans):
    B, od, G, H, W, P, part, S, ncls = case
    if no_trans:
        ncls = 1
    gen = _gen(case, no_trans)
    C = od * G * G
    data = torch.randn(B, C, H, W, generator=gen)
    rois = R.edge_rois(H, W, B, P, S, 24, gen)
    N = rois.shape[0]
    trans = (torch.randn(N, 2 * ncls, part, part, generator=gen) * 1.5)
    kw = dict(spatial_scale=0.0625, output_dim=od, group_size=G, trans_std=0.1)
    out, cnt, sidx = O.deform_psroi_fwd(data.numpy(), rois.numpy(), trans.numpy(), pooled=P, part_size=part, spp=S,
                                        no_trans=no_trans, **kw)
    g = R.ps_geom(rois, None if no_trans else trans, H=H, W=W, spatial_scale=0.0625, pooled=P, part_size=part,
                  sample_per_part=S, trans_std=0.1, no_trans=no_trans, ncls=ncls)
    ce = od // ncls
    assert np.array_equal(R.ps_sample_idx(g, W, od, ce).numpy(), sidx)
    rc = R.ps_count(g)[:, torch.arange(od) // ce].float().numpy()
    assert np.array_equal(rc, cnt)
    assert (cnt == 0).any() and (cnt == S * S).any() and (S == 1 or ((cnt > 0) & (cnt < S * S)).any())
    ref, mag = R.deform_psroi_fwd(data.double(), g, output_dim=od, group_size=G)
    err = np.abs(out - ref.numpy())
    assert (err <= (S * S + 8) * U * 1.01 * mag.numpy() + 1e-30).all(), err.max()
    assert (out[cnt == 0] == 0).all()
    # gradients: the oracle accumulates float32 terms in double
    td = torch.randn(N, od, P, P, generator=gen)
    dd, tdd = O.deform_psroi_bwd(td.numpy(), cnt, data.numpy(), rois.numpy(), trans.numpy(), pooled=P, part_size=part,
                                 spp=S, no_trans=no_trans, **kw)
    G64 = R.deform_psroi_bwd(td, data.double(), g, output_dim=od, group_size=G, trans_std=0.1, no_trans=no_trans)
    e = np.abs(dd - G64["data_diff"].numpy())
    assert (e <= 5 * U * 1.01 * G64["dd_mag"].numpy() + 1e-300).all(), e.max()
    if not no_trans:
        e = np.abs(tdd - G64["trans_diff"].numpy())
        assert (e <= 10 * U * 1.01 * G64["td_mag"].numpy() + 1e-300).all(), e.max()
        assert (tdd[G64["td_bins"].numpy() == 0] == 0).all()


@pytest.mark.parametrize("case", [(2, 2, 3, 20, 24, 3), (2, 1, 7, 1, 13, 7), (3, 4, 1, 9, 30, 7)],
                         ids=lambda c: "B%d-od%d-g%d-%dx%d-P%d" % c)
def test_psroi_reference_against_oracle(case):
    B, od, G, H, W, P = case
    gen = _gen("psroi", case)
    data = torch.randn(B, od * G * G, H, W, generator=gen)
    rois = R.edge_rois(H, W, B, P, 1, 24, gen)
    out, bins = O.psroi_fwd(data.numpy(), rois.numpy(), 0.0625, od, G, P)
    rb = R.psroi_bins(rois, H=H, W=W, spatial_scale=0.0625, pooled=P)
    assert np.array_equal(R.psroi_bins_array(rb, od).numpy(), bins)
    ref, mag = R.psroi_fwd(data, rb, output_dim=od, group_size=G)
    area = (bins[:, 1] - bins[:, 0]) * (bins[:, 3] - bins[:, 2])
    k = np.maximum(area, 1).reshape(out.shape) + 1
    assert (np.abs(out - ref.numpy()) <= k * U * 1.01 * mag.numpy() + 1e-12 * float(mag.max())).all()
    td = torch.randn(*out.shape, generator=gen)
    dd = O.psroi_bwd(td.numpy(), rois.numpy(), data.shape, 0.0625, od, G, P)
    ref_dd, ref_mag, terms = R.psroi_bwd(td, rb, data.shape, output_dim=od, group_size=G)
    e = np.abs(dd - ref_dd.numpy())
    # the float64 prefix sums of the reference carry ~1e-16 of the plane's total: 1e-12 * max|terms| absolute
    assert (e <= 1.01 * U * ref_mag.numpy() + 1e-12 * float(ref_mag.max())).all(), e.max()
    assert (dd[terms.numpy() == 0] == 0).all()


def test_deform_conv_reference_against_graph_oracle():
    import torch_graph as TG
    gen = _gen("dc-graph")
    N, C, H, W, dg = 2, 256, 9, 13, 2
    x = torch.randn(N, C, H, W, generator=gen, dtype=torch.float64)
    off = torch.round(torch.randn(N, dg * 18, H, W, generator=gen, dtype=torch.float64) * 2 * 1024) / 1024
    off[:, :, 0, :4] = torch.tensor([-2.0, 0.0, 2.0, 9.0], dtype=torch.float64)   # whole-pixel and far-out samples
    w = torch.randn(16, C, 3, 3, generator=gen, dtype=torch.float64)
    TG.MODE[0] = "exact"
    y = TG.deform_conv2d(x, off, w, dil=2, pad=2, dg=dg)                        # [N, 16, H, W]
    col, _ = R.dc_im2col(x.permute(0, 2, 3, 1).contiguous(), off.permute(0, 2, 3, 1).float().contiguous(), 3, 3, 1, 2,
                         2, dg)
    y2 = col @ w.permute(0, 2, 3, 1).reshape(16, 9 * C).t()
    y2 = y2.view(N, H, W, 16).permute(0, 3, 1, 2)
    assert float((y - y2).abs().max()) <= 1e-12 * float(y.abs().max())


def test_deform_conv_geometry_edges():
    """h_im on -1, -2^-20, 0, 0.5, H-1-2^-20, H-1, H-0.5, H-2^-20, H: validity and clamps as the kernel's rules say"""
    H = W = 6
    vals = [-1.0, -2.0 ** -20, 0.0, 0.5, H - 1 - 2.0 ** -20, H - 1.0, H - 0.5, H - 2.0 ** -20, float(H)]
    # one tap (1x1 kernel, pad 0): h_im = ho + off_h, w_im = wo + off_w; put every value at output (0, 0)
    off = torch.zeros(len(vals), 1, 1, 2)
    off[:, 0, 0, 0] = torch.tensor(vals)
    x = torch.randn(len(vals), H, W, 128, dtype=torch.float64)
    col, _ = R.dc_im2col(x, off.reshape(len(vals), 1, 1, 2).expand(len(vals), H, W, 2).contiguous(), 1, 1, 1, 1, 0, 1)
    col = col.view(len(vals), H, W, 128)[:, 0, 0]
    for k, v in enumerate(vals):
        if v < 0 or v >= H:
            assert (col[k] == 0).all(), v
        else:
            lo = min(int(np.floor(v)), H - 1)
            f = 0.0 if np.floor(v) >= H - 1 else float(np.float32(v)) - lo
            exp = (1 - f) * x[k, lo, 0] + (f * x[k, lo + 1, 0] if f else 0)
            assert torch.allclose(col[k], exp, rtol=0, atol=1e-12), v


def test_deform_conv_gradients_against_central_differences():
    gen = _gen("dc-fd")
    NB, H, W, C, dg, KH, KW, st, dil, pad = 2, 7, 9, 256, 2, 3, 3, 2, 1, 1
    Ho, Wo = R.out_extent(H, KH, st, dil, pad), R.out_extent(W, KW, st, dil, pad)
    x = torch.randn(NB, H, W, C, generator=gen, dtype=torch.float64)
    # fractions in [0.25, 0.75]: a step of 1e-4 never crosses a pixel boundary
    off = (torch.randint(-2, 2, (NB, Ho, Wo, dg * 2 * 9), generator=gen) + 0.25 +
           0.5 * torch.rand(NB, Ho, Wo, dg * 2 * 9, generator=gen)).float()
    dcol = torch.randn(NB * Ho * Wo, 9 * C, generator=gen, dtype=torch.float64)
    G = R.dc_col2im(dcol, x, off, KH, KW, st, dil, pad, dg)
    f = lambda xx, oo: float((R.dc_im2col(xx, oo, KH, KW, st, dil, pad, dg)[0] * dcol).sum())
    h = 2.0 ** -12
    for (n, i, j, k) in [(0, 1, 2, 3), (1, 2, 0, 20), (1, Ho - 1, Wo - 1, 35), (0, 0, 0, 33)]:
        op, om = off.clone(), off.clone()
        op[n, i, j, k] += h
        om[n, i, j, k] -= h
        fd = (f(x, op) - f(x, om)) / (2 * h)
        assert abs(fd - float(G["doff"][n, i, j, k])) <= 1e-6 * (1 + abs(fd)), (n, i, j, k)
    for (n, i, j, c) in [(0, 3, 4, 5), (1, 0, 0, 200), (1, 6, 8, 130)]:
        xp, xm = x.clone(), x.clone()
        xp[n, i, j, c] += 1e-3
        xm[n, i, j, c] -= 1e-3
        fd = (f(xp, off) - f(xm, off)) / 2e-3
        assert abs(fd - float(G["dx"][n, i, j, c])) <= 1e-8 * (1 + abs(fd))


def test_deform_psroi_gradients_against_central_differences():
    gen = _gen("ps-fd")
    B, od, H, W, P, S = 2, 4, 12, 16, 3, 2
    data = torch.randn(B, od, H, W, generator=gen, dtype=torch.float64)
    rois = torch.tensor([[0, 16, 16, 150, 120], [1, 40, 8, 200, 180]], dtype=torch.float32)
    trans = (torch.rand(2, 2, P, P, generator=gen) * 0.5 - 0.25).float()
    td = torch.randn(2, od, P, P, generator=gen)
    kw = dict(H=H, W=W, spatial_scale=0.0625, pooled=P, part_size=P, sample_per_part=S, trans_std=0.1, no_trans=False,
              ncls=1)
    G = R.deform_psroi_bwd(td, data, R.ps_geom(rois, trans, **kw), output_dim=od, group_size=1, trans_std=0.1,
                           no_trans=False)

    def f(d, t):
        return float((R.deform_psroi_fwd(d, R.ps_geom(rois, t, **kw), output_dim=od, group_size=1)[0] * td.double()).sum())
    h = 2.0 ** -10
    for idx in [(0, 0, 1, 1), (1, 1, 0, 2), (0, 1, 2, 0)]:
        tp, tm = trans.clone(), trans.clone()
        tp[idx] += h
        tm[idx] -= h
        fd = (f(data, tp) - f(data, tm)) / (2 * h)
        # the float32 sample positions move by steps of their own ulp: a few 1e-6 of slack
        assert abs(fd - float(G["trans_diff"][idx])) <= 2e-4 * (1 + abs(fd)), idx
    for idx in [(0, 1, 3, 3), (1, 2, 5, 7)]:
        dp, dm = data.clone(), data.clone()
        dp[idx] += 1e-3
        dm[idx] -= 1e-3
        fd = (f(dp, trans) - f(dm, trans)) / 2e-3
        assert abs(fd - float(G["data_diff"][idx])) <= 1e-9 * (1 + abs(fd))
