"""The depthwise 3x3 weight gradient (sniper_depthwise3x3_wgrad) against float64, and its reproducibility.

The kernel sums block partials in a fixed order through a caller-owned workspace, so two launches must give the same
bits, eagerly and under CUDA-graph capture and replay.  Cases: fp32 and bf16, stride 1 and 2; every (C, H, W,
stride) of the 17 inverted-residual units of MobileNetV2 at B = 40 on 512 x 512 chips (channels padded to 64 as the
network stores them); ragged maps; channel counts on the LC = 16 lane path (64, 192) and the LC = 32 path (128, 384);
accumulation into a non-zero dw; NaN guard regions around dw that must stay untouched.

Error bound.  Every output is a float32 sum of N = NB * Ho * Wo products (bf16 products are exact in float32, float32
products round once).  Its additions form a tree of depth at most
    d = (strips per thread) * PW + 8 * 32 / LC   (thread, then the shared-memory strip reduction)
        + ceil(gx / 8) + 8 + 1                    (the fixed-order slab reduction, then the one addition into dw),
so |got - exact| <= (d + 1) * 2^-24 * (sum |products| + |dw0|) + 2^-24 * |exact|.  The grid gx is not visible from
here; the bound takes the smallest gx the one-wave rule can pick (one block per SM) for the per-thread depth and the
largest for the slab depth.  Seeds come from the crc32 of the case id, so a failure reproduces."""
import os
import sys
import zlib

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
SMS, SLAB_FLOATS = 132, 132 * 4 * 9 * 128
U = 2.0 ** -24


def _seed(*key):
    return zlib.crc32(repr(key).encode())


def _unit_shapes(B=40, chip=512):
    """(NB, H, W, C, stride) of the depthwise layer of each inverted-residual unit (model_mnv2.MCfg.bottlenecks)."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from sniper_b200 import model_mnv2 as MM
    cfg = MM.MCfg()
    H = (chip - 1) // 2 + 1                      # first 3x3 / stride 2 conv
    out, cin = [], cfg.first_c
    for t, c, n, s in cfg.bottlenecks:
        for j in range(n):
            e = int(round((cin if j == 0 else c) * t))
            st = s if j == 0 else 1
            out.append((B, H, H, MM.pad64(e), st))
            H = (H - 1) // st + 1
        cin = c
    return out


UNITS = _unit_shapes()
assert len(UNITS) == 17
OTHER = [(3, 17, 23, 192, 1), (2, 15, 9, 64, 2), (1, 1, 1, 64, 1), (2, 7, 5, 8, 2), (4, 33, 31, 128, 2),
         (2, 16, 16, 384, 1), (1, 3, 130, 192, 2), (2, 64, 64, 960, 1)]
CASES = [("unit%02d" % i, ) + u for i, u in enumerate(UNITS)] + [("ragged%d" % i, ) + o for i, o in enumerate(OTHER)]


def _inputs(NB, H, W, C, stride, dt, g):
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    x = torch.randn(NB, H, W, C, device=DEV, generator=g).to(dt)
    dy = torch.randn(NB, Ho, Wo, C, device=DEV, generator=g).to(dt)
    return x, dy


def _ref(x, dy, stride):
    """float64 sum of dy * shifted x per (tap, channel), and the sum of the products' magnitudes."""
    NB, H, W, C = x.shape
    _, Ho, Wo, _ = dy.shape
    xp = torch.nn.functional.pad(x.double(), (0, 0, 1, 1, 1, 1))
    d = dy.double()
    ref = torch.empty(9, C, dtype=torch.float64, device=DEV)
    mag = torch.empty(9, C, dtype=torch.float64, device=DEV)
    for kh in range(3):
        for kw in range(3):
            xs = xp[:, kh:kh + (Ho - 1) * stride + 1:stride, kw:kw + (Wo - 1) * stride + 1:stride]
            prod = xs * d
            ref[kh * 3 + kw] = prod.sum((0, 1, 2))
            mag[kh * 3 + kw] = prod.abs().sum((0, 1, 2))
            del prod
    return ref, mag


def _depth(NB, H, W, C, stride):
    PW = 4 if stride == 1 else 2
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    LC = 32 if (C // 4) % 32 == 0 else 16
    PL = 8 * (32 // LC)
    gy = -(-(C // 4) // LC)
    strips = NB * Ho * -(-Wo // PW)
    gx_cap = min(-(-strips // PL), SLAB_FLOATS // (9 * C))
    gx_lo = max(1, min(gx_cap, SMS // gy))
    gx_hi = max(1, gx_cap)
    per_thread = -(-strips // (gx_lo * PL))
    return per_thread * PW + 8 * (32 // LC) + -(-gx_hi // 8) + 8 + 1


def _guarded(C, dw0):
    """dw [9, C] inside a NaN-filled buffer: 64 floats of guard before and after."""
    buf = torch.full((9 * C + 128, ), float("nan"), device=DEV)
    dw = buf[64:64 + 9 * C].view(9, C)
    dw.copy_(dw0)
    return buf, dw


def _check_guards(buf, C):
    assert torch.isnan(buf[:64]).all() and torch.isnan(buf[64 + 9 * C:]).all(), "wrote outside dw"


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_wgrad_matches_float64_and_reproduces(case, dtype):
    from sniper_b200 import ops
    name, (NB, H, W, C, stride) = case[0], case[1:]
    dt = torch.float32 if dtype == "fp32" else torch.bfloat16
    g = torch.Generator(device=DEV)
    g.manual_seed(_seed(name, dtype))
    x, dy = _inputs(NB, H, W, C, stride, dt, g)
    dw0 = torch.randn(9, C, device=DEV, generator=g) * 4.0        # accumulate into a non-zero dw
    ref, mag = _ref(x, dy, stride)
    buf, dw = _guarded(C, dw0)
    ops.depthwise3x3_wgrad(x, dy, dw, stride)
    torch.cuda.synchronize()
    _check_guards(buf, C)
    exact = dw0.double() + ref
    err = (dw.double() - exact).abs()
    d = _depth(NB, H, W, C, stride)
    bound = (d + 1) * U * (mag + dw0.double().abs()) + U * exact.abs()
    ratio = (err / bound).max().item()
    print("%s %s C=%d %dx%d s%d: depth %d, worst err/bound %.3g" % (name, dtype, C, H, W, stride, d, ratio))
    assert ratio <= 1.0, (name, dtype, ratio)
    # a second eager launch: the same bits
    buf2, dw2 = _guarded(C, dw0)
    ops.depthwise3x3_wgrad(x, dy, dw2, stride)
    torch.cuda.synchronize()
    _check_guards(buf2, C)
    assert torch.equal(dw2.view(torch.int32), dw.view(torch.int32)), "two eager launches differ"


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("case", [CASES[0], CASES[1], CASES[16], CASES[17], CASES[20]], ids=lambda c: c[0])
def test_wgrad_graph_replay_is_byte_identical_to_eager(case, dtype):
    from sniper_b200 import ops
    name, (NB, H, W, C, stride) = case[0], case[1:]
    dt = torch.float32 if dtype == "fp32" else torch.bfloat16
    g = torch.Generator(device=DEV)
    g.manual_seed(_seed(name, dtype, "graph"))
    x, dy = _inputs(NB, H, W, C, stride, dt, g)
    dw0 = torch.randn(9, C, device=DEV, generator=g)
    buf, dw = _guarded(C, dw0)
    ops.depthwise3x3_wgrad(x, dy, dw, stride)
    torch.cuda.synchronize()
    eager = dw.clone()
    gbuf, gdw = _guarded(C, dw0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.depthwise3x3_wgrad(x, dy, gdw, stride)
    for i in range(3):
        gdw.copy_(dw0)
        graph.replay()
        torch.cuda.synchronize()
        _check_guards(gbuf, C)
        assert torch.equal(gdw.view(torch.int32), eager.view(torch.int32)), "replay %d differs from eager" % i
    # eager launches on two streams at once use separate workspaces
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = []
    torch.cuda.synchronize()
    for s in (s1, s2):
        with torch.cuda.stream(s):
            b, d = _guarded(C, dw0)
            ops.depthwise3x3_wgrad(x, dy, d, stride)
            outs.append((b, d))
    torch.cuda.synchronize()
    for b, d in outs:
        _check_guards(b, C)
        assert torch.equal(d.view(torch.int32), eager.view(torch.int32)), "concurrent streams differ"
