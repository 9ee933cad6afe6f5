"""The tf32 weight gradient's operand copy area (csrc/gemm_tc.cu, WgradFeed), host only.

For stride-1 layers with several taps over rows of Wo % 32 == 0 pixels, sniper_conv2d_wgrad_nhwc copies dY and X
channel-major into the copy area of the stream's workspace before its K-major mainloop; other layers and bf16 need
none.  sniper_conv2d_wgrad_scratch_bytes must give the size of that layout for a geometry, restated here in Python: dY^T
[Cout, P] with P = NB * Ho * Wo, its row pitch rounded up to 16 bytes, then at the next 256-byte boundary X^T
[cols * Cin, NB * Hp * Wo], one block of Cin rows per distinct column offset dw of the taps, over the input rows
zero-padded to Hp.
"""
import ctypes
import os
import sys

import numpy as np
import pytest

from sniper_b200 import _lib, ops

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gemm_exact_gpu as X  # noqa: E402


def _round(v, m):
    return -(-v // m) * m


def expected_bytes(NB, H, W, Cin, Cout, dh, dw, stride, Ho, Wo):
    """(layout, bytes) by the rule above"""
    ntaps = len(dh)
    P = NB * Ho * Wo
    if ntaps == 1 or stride != 1 or Wo % 32:
        return "none", 0
    Hp = H + max([0] + [-d for d in dh]) + max([0] + [Ho - 1 + d - (H - 1) for d in dh])
    layout, rows, pixels = "copies", len(set(dw)) * Cin, NB * Hp * Wo
    return layout, _round(Cout * _round(P, 4) * 4, 256) + rows * _round(pixels, 4) * 4


def query(NB, H, W, Cin, Cout, dh, dw, stride, Ho, Wo, dtype=0):
    a = np.ascontiguousarray(dh, dtype=np.int32)
    b = np.ascontiguousarray(dw, dtype=np.int32)
    return _lib.lib().sniper_conv2d_wgrad_scratch_bytes(NB, H, W, Cin, Cout, len(dh), a.ctypes.data_as(ctypes.c_void_p),
                                                        b.ctypes.data_as(ctypes.c_void_p), stride, Ho, Wo, dtype)


def geometry(NB, H, W, Cin, Cout, k, stride=1, dil=1, pad=0):
    dh, dw = ops.conv_taps(k, k, dil, pad)
    Ho = (H + 2 * pad - dil * (k - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (k - 1) - 1) // stride + 1
    return NB, H, W, Cin, Cout, dh, dw, stride, Ho, Wo


# Weight gradients of the ResNet-101 step at 20 chips of 512 x 512 (stages at 128 / 64 / 32 / 32 pixels), the R-FCN
# head's fc_new_1, and MobileNetV2's RPN 3 x 3 on the stride-32 map: (id, geometry, layout)
STEP = [
    ("stage2_unit1_conv1", geometry(20, 128, 128, 256, 128, 1), "none"),
    ("stage2_unit1_conv2_s2", geometry(20, 128, 128, 128, 128, 3, stride=2, pad=1), "none"),
    ("stage2_unit1_sc_s2", geometry(20, 128, 128, 256, 512, 1, stride=2), "none"),
    ("stage3_conv2", geometry(20, 32, 32, 256, 256, 3, pad=1), "copies"),
    ("stage4_conv2_dil2", geometry(20, 32, 32, 512, 512, 3, dil=2, pad=2), "copies"),
    ("rpn_conv_3x3", geometry(20, 32, 32, 3072, 512, 3, pad=1), "copies"),
    ("fc_new_1", (1, 1, 6000, 12544, 1024, [0], [0], 1, 1, 6000), "none"),
    ("mnv2_rpn_conv_3x3_wo16", geometry(20, 16, 16, 1280, 256, 3, pad=1), "none"),
]


@pytest.mark.parametrize("case", STEP, ids=lambda c: c[0])
def test_scratch_bytes_of_the_step(case):
    cid, g, layout = case
    want_layout, want = expected_bytes(*g)
    assert want_layout == layout, cid
    assert query(*g) == want, cid
    assert query(*g, dtype=1) == 0, cid


def test_padded_extent_of_a_3x3_layer():
    """stage-3 conv2: 3 column offsets x 256 channels over 20 x 34 x 32 pixels (one zero row above and below)"""
    assert query(*STEP[3][1]) == 256 * 20 * 32 * 32 * 4 + 3 * 256 * 20 * 34 * 32 * 4


def test_largest_step_call():
    """rpn_conv_3x3: dY^T 512 x 20480 and X^T 3 x 3072 rows over 20 x 34 x 32 pixels, fp32 (0.84 GB)"""
    assert query(*STEP[5][1]) == 512 * 20480 * 4 + 3 * 3072 * 20 * 34 * 32 * 4


@pytest.mark.parametrize("w", X.WGRAD, ids=lambda w: w.id)
def test_scratch_bytes_of_the_exact_table(w):
    for dt, dtype in (("tf32", 0), ("bf16", 1)):
        g = geometry(w.NB, w.H, w.W, w.Cin, X.wgrad_cout(w, dt), w.k, w.stride, w.dil, w.pad)
        if w.id == "fc_new_1":
            g = (1, 1, w.W, w.Cin, X.wgrad_cout(w, dt), [0], [0], 1, 1, w.W)
        got = query(*g, dtype=dtype)
        assert got == (expected_bytes(*g)[1] if dt == "tf32" else 0), (w.id, dt)


def test_exact_table_covers_every_layout():
    layouts = set()
    for w in X.WGRAD:
        g = geometry(w.NB, w.H, w.W, w.Cin, 96, w.k, w.stride, w.dil, w.pad)
        if w.id == "fc_new_1":
            g = (1, 1, w.W, w.Cin, 1024, [0], [0], 1, 1, w.W)
        layouts.add(expected_bytes(*g)[0])
    assert layouts == {"none", "copies"}


def test_ragged_pitch_rounds_to_16_bytes():
    """3 x 3 over 1 x 3 x 32: P = 96; dY^T 33 x 96 floats is rounded up to 256 bytes, X^T 3 x 64 rows of 5 x 32"""
    g = geometry(1, 3, 32, 64, 33, 3, pad=1)
    assert query(*g) == _round(33 * 96 * 4, 256) + 3 * 64 * 160 * 4
