"""The case tables of test_gemm_exact_gpu.py reach the wgmma instantiations they claim (host only, no GPU).

`sniper_gemm_plan` gives the tile width and the tail split sniper_gemm_nt would choose; a convolution is planned as the
GEMM of its kernel rows (M' = NB * tiles_per_img * 128, N = Cout, K = taps * Cin).  Without this check a shape change
could silently move an exact case off the path it is meant to cover.  Weight-gradient rows have no plan query: their
tile arithmetic is stated in the row comments and restated by `wgrad_tiles`.
"""
import ctypes
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gemm_exact_gpu as X  # noqa: E402

# every gemm_tc_kernel<DT, MN, BN, PN> that launch() can pick
ALL_INSTANTIATIONS = ({(dt, 0, bn, 0) for dt in X.DTS for bn in (64, 128, 256)} |
                      {(dt, 0, 256, pn) for dt in X.DTS for pn in (64, 128)} |
                      {(dt, 1, bn, 0) for dt in X.DTS for bn in (64, 128, 256)})


def _plan(M, N, K, dt):
    from sniper_b200 import _lib
    out = (ctypes.c_int * 8)()
    _lib.check(_lib.lib().sniper_gemm_plan(M, N, K, 0 if dt == "tf32" else 1, ctypes.cast(out, ctypes.c_void_p)))
    bn, _, _, tiles, _, mode, _, pieces = list(out)
    return bn, mode, pieces, tiles


def _kmajor_shapes():
    """(id, claimed inst, dt, M', N, K) of every K-major row: GEMMs, convolutions and the stride-2 data gradients"""
    for c in X.GEMM:
        for dt in X.DTS:
            yield c.id, c.inst, dt, c.M, c.N, c.kb * X.E[dt]
    for c in X.CONV:
        Ho, Wo = X.conv_out_hw(c)
        for dt in X.DTS:
            yield c.id, c.inst, dt, X.conv_rows(c.NB, Ho, Wo), c.Cout, c.k * c.k * c.Cin
    for c in X.DGRAD:
        for dt in X.DTS:      # every parity-class conv runs over the H/2 x W/2 grid with N = cin; K does not matter here
            yield c.id, c.inst, dt, X.conv_rows(c.NB, c.H // 2, c.W // 2), c.cin, c.cout


def test_case_table_reaches_all_16_instantiations():
    claimed = {(dt,) + tuple(c.inst) for rows in (X.GEMM, X.CONV, X.DGRAD, X.WGRAD) for c in rows for dt in X.DTS}
    assert claimed == ALL_INSTANTIATIONS, sorted(ALL_INSTANTIATIONS - claimed)
    print("reached:", ", ".join("<%s,%d,%d,%d>" % i for i in sorted(claimed)))
    # several work units per CTA (132 persistent CTAs): a K-major case of each width, and a weight gradient
    for bn in (64, 128, 256):
        assert any(_plan(c.M, c.N, c.kb * X.E["tf32"], "tf32")[3] > 132 for c in X.GEMM
                   if c.inst == (0, bn, 0)), bn
    assert any(X.wgrad_tiles(w, dt) > 132 for w in X.WGRAD for dt in X.DTS)


@pytest.mark.parametrize("case", list(_kmajor_shapes()), ids=lambda c: "%s-%s" % (c[0], c[2]))
def test_kmajor_case_takes_its_claimed_path(case):
    cid, (mn, bn, pn), dt, M, N, K = case
    assert mn == 0
    got_bn, mode, pieces, _ = _plan(M, N, K, dt)
    want = (bn, 2, bn // pn) if pn else (bn, 0, 1)
    assert (got_bn, mode, pieces) == want, (cid, dt, M, N, K)


def test_wgrad_rows_tile_arithmetic():
    """The row comments' arithmetic: BN from Cin, and the tile counts quoted there.  This is a restatement of the width
    rule of sniper_conv2d_wgrad_nhwc in Python, not a query of the C code (there is no plan entry point for weight
    gradients): a change to that rule does not move this test, unlike the sniper_gemm_plan checks above."""
    for w in X.WGRAD:
        bn = 256 if w.Cin % 256 == 0 else (128 if w.Cin % 128 == 0 else 64)
        assert w.inst == (1, bn, 0), w.id
    fc = [w for w in X.WGRAD if w.id == "fc_new_1"][0]
    assert X.wgrad_tiles(fc, "tf32") == X.wgrad_tiles(fc, "bf16") == 392
