"""GPU parity: (Deformable)PSROIPooling vs the CPU oracle."""
import numpy as np
import pytest

import oracle_lib as O
from sniper_b200 import synth

pytestmark = pytest.mark.gpu


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("no_trans", [True, False])
@pytest.mark.parametrize("layout", [0, 1])
def test_deform_psroi_reference_test_shape(no_trans, layout):
    # shapes/params of the reference's own test (test_operator.py:4358-4389)
    from sniper_b200 import ops
    rng = np.random.RandomState(3)
    data = rng.rand(2, 18, 14, 14).astype(np.float32)
    rois = np.array([[0, 10, 22, 161, 173], [1, 20, 15, 154, 160], [0, 0, 0, 5, 5], [1, 100, 100, 400, 300]], np.float32)
    trans = (rng.rand(4, 4, 3, 3).astype(np.float32) - 0.5)
    kw = dict(spatial_scale=0.0625, output_dim=2, group_size=3, trans_std=0.1)
    out, cnt, sidx = O.deform_psroi_fwd(data, rois, trans, pooled=3, part_size=3, spp=4, no_trans=no_trans, **kw)
    d = _t(data if layout == 0 else data.transpose(0, 2, 3, 1))
    g_out, g_cnt, g_sidx = ops.deform_psroi_fwd(d, _t(rois), _t(trans), pooled_size=3, part_size=3, sample_per_part=4,
                                               no_trans=no_trans, layout=layout, want_sample_idx=True, **kw)
    g_out, g_cnt = g_out.cpu().numpy(), g_cnt.cpu().numpy()
    if layout == 1:
        g_out, g_cnt = g_out.transpose(0, 3, 1, 2), g_cnt.transpose(0, 3, 1, 2)
    np.testing.assert_array_equal(g_sidx.cpu().numpy(), sidx)       # ROI sample indices: bit-exact
    np.testing.assert_array_equal(g_cnt, cnt)
    assert g_out.tobytes() == np.ascontiguousarray(out).tobytes()   # same op order -> same bits
    # backward
    g = rng.randn(*out.shape).astype(np.float32)
    dd, td = O.deform_psroi_bwd(g, cnt, data, rois, trans, pooled=3, part_size=3, spp=4, no_trans=no_trans, **kw)
    gt = _t(g if layout == 0 else g.transpose(0, 2, 3, 1))
    g_dd, g_td = ops.deform_psroi_bwd(gt, d, _t(rois), _t(trans), pooled_size=3, part_size=3, sample_per_part=4,
                                      no_trans=no_trans, layout=layout, **kw)
    g_dd = g_dd.cpu().numpy()
    if layout == 1:
        g_dd = g_dd.transpose(0, 3, 1, 2)
    np.testing.assert_allclose(g_dd, dd, rtol=1e-4, atol=1e-5)
    if not no_trans:
        np.testing.assert_allclose(g_td.cpu().numpy(), td, rtol=1e-3, atol=1e-4)


def test_deform_psroi_sniper_shape():
    # the two calls of the ResNet-101 head (resnet_mx_101_e2e.py:286-293): 256 ch, 7x7, 4x4 samples, 1/16
    from sniper_b200 import ops
    rng = np.random.RandomState(7)
    B, C = 3, 256
    data = rng.randn(B, C, 32, 32).astype(np.float32)
    rois = synth.rois_for_pool(rng, 200, B)
    trans = (rng.randn(200, 2, 7, 7) * 0.5).astype(np.float32)
    kw = dict(spatial_scale=0.0625, output_dim=256, group_size=1, trans_std=0.1)
    for no_trans in (True, False):
        out, cnt, sidx = O.deform_psroi_fwd(data, rois, trans, pooled=7, part_size=7, spp=4, no_trans=no_trans, **kw)
        for layout in (0, 1):
            d = _t(data if layout == 0 else data.transpose(0, 2, 3, 1))
            g_out, g_cnt, g_sidx = ops.deform_psroi_fwd(d, _t(rois), _t(trans), pooled_size=7, part_size=7,
                                                       sample_per_part=4, no_trans=no_trans, layout=layout,
                                                       want_sample_idx=True, **kw)
            g_out, g_cnt = g_out.cpu().numpy(), g_cnt.cpu().numpy()
            if layout == 1:
                g_out, g_cnt = g_out.transpose(0, 3, 1, 2), g_cnt.transpose(0, 3, 1, 2)
            np.testing.assert_array_equal(g_sidx.cpu().numpy(), sidx)
            np.testing.assert_array_equal(g_cnt, cnt)
            assert g_out.tobytes() == np.ascontiguousarray(out).tobytes()
            if layout == 1:
                import os
                # warp-per-bin kernels (taken when no sample indices are requested).  SNIPER_PSROI_EXACT=1: per-sample
                # operation order of the oracle -> same bits; default: separable form (each touched pixel gathered
                # once with the summed weight) -> same counts, values to fp32 rounding (tolerance 2e-6 * max|data|).
                os.environ["SNIPER_PSROI_EXACT"] = "1"
                try:
                    f_out, f_cnt, _ = ops.deform_psroi_fwd(d, _t(rois), _t(trans), pooled_size=7, part_size=7,
                                                           sample_per_part=4, no_trans=no_trans, layout=1, **kw)
                finally:
                    os.environ.pop("SNIPER_PSROI_EXACT", None)
                assert f_out.cpu().numpy().transpose(0, 3, 1, 2).tobytes() == g_out.tobytes()
                np.testing.assert_array_equal(f_cnt.cpu().numpy().transpose(0, 3, 1, 2), cnt)
                s_out, s_cnt, _ = ops.deform_psroi_fwd(d, _t(rois), _t(trans), pooled_size=7, part_size=7,
                                                       sample_per_part=4, no_trans=no_trans, layout=1, **kw)
                np.testing.assert_array_equal(s_cnt.cpu().numpy().transpose(0, 3, 1, 2), cnt)
                err = np.abs(s_out.cpu().numpy().transpose(0, 3, 1, 2) - out).max()
                assert err <= 2e-6 * np.abs(data).max(), err
    g = rng.randn(200, 256, 7, 7).astype(np.float32)
    dd, td = O.deform_psroi_bwd(g, cnt, data, rois, trans, pooled=7, part_size=7, spp=4, no_trans=False, **kw)
    g_dd, g_td = ops.deform_psroi_bwd(_t(g.transpose(0, 2, 3, 1)), _t(data.transpose(0, 2, 3, 1)), _t(rois), _t(trans),
                                      pooled_size=7, part_size=7, sample_per_part=4, no_trans=False, layout=1, **kw)
    np.testing.assert_allclose(g_dd.cpu().numpy().transpose(0, 3, 1, 2), dd, rtol=2e-4, atol=2e-4)
    np.testing.assert_allclose(g_td.cpu().numpy(), td, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("layout", [0, 1])
def test_psroi(layout):
    from sniper_b200 import ops
    rng = np.random.RandomState(9)
    data = rng.randn(2, 2 * 9, 20, 24).astype(np.float32)
    rois = synth.rois_for_pool(rng, 64, 2, chip=320)
    rois[0, 1:] = (5, 5, 5, 5)      # degenerate roi
    rois[1, 1:] = (300, 300, 319, 319)
    out, bins = O.psroi_fwd(data, rois, 0.0625, 2, 3, 3)
    d = _t(data if layout == 0 else data.transpose(0, 2, 3, 1))
    g_out, g_bins = ops.psroi_fwd(d, _t(rois), spatial_scale=0.0625, output_dim=2, group_size=3, pooled_size=3,
                                  layout=layout, want_bins=True)
    np.testing.assert_array_equal(g_bins.cpu().numpy(), bins)       # ROI bin indices: bit-exact
    g_out = g_out.cpu().numpy()
    if layout == 1:
        g_out = g_out.transpose(0, 3, 1, 2)
    assert g_out.tobytes() == np.ascontiguousarray(out).tobytes()
    g = rng.randn(*out.shape).astype(np.float32)
    dd = O.psroi_bwd(g, rois, data.shape, 0.0625, 2, 3, 3)
    shape = data.shape if layout == 0 else (2, 20, 24, 18)
    gt = _t(g if layout == 0 else g.transpose(0, 2, 3, 1))
    g_dd = ops.psroi_bwd(gt, _t(rois), shape, spatial_scale=0.0625, output_dim=2, group_size=3, pooled_size=3,
                         layout=layout).cpu().numpy()
    if layout == 1:
        g_dd = g_dd.transpose(0, 3, 1, 2)
    np.testing.assert_allclose(g_dd, dd, rtol=1e-4, atol=1e-5)
