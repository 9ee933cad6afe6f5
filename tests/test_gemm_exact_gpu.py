"""Every instantiation of the wgmma kernel (gemm_tc.cu) and every launch path, compared BIT FOR BIT with float64.

Operands are random integers in {-1, 0, 1}; biases and residuals are small integers and scales are powers of two.  The
products are then exact in TF32 and bf16, and every partial sum the kernel can form (any K order, any split-K order,
fp32 atomics, the double atomics of the fused statistics) is an integer below 2^24, so the result does not depend on
summation order: it must equal the float64 reference exactly.  One missing, duplicated or misplaced product term moves
an output by at least 1.  `_check_range` asserts that precondition on the reference before each comparison.

The case tables are plain data at module level (no device work at import): tests/test_gemm_exact_cpu.py checks on the
host that each row reaches the instantiation `(dt, mn, bn, pn)` it names.  Every row runs for tf32 and bf16.  K-major
rows give K in k-blocks (kb): K = kb * 32 (tf32) or kb * 64 (bf16) elements.  Ring depths (pick_stages): K-major 8 / 6 / 4
stages for BN 64 / 128 / 256; weight gradients 6 / 4 / 2 (tf32, two stages go to the K-major transpose ring) and
8 / 6 / 4 (bf16).  132 persistent CTAs; column pieces when the last wave holds 1..66 tiles of a 256-wide N > 256
problem: 4 x 64 columns for up to 33 tail tiles, else 2 x 128.

The second half checks the operand rounding of each operand path on random data, where the exact cases are blind.
"""
import collections

import pytest
import torch

pytestmark = pytest.mark.gpu

DTS = ("tf32", "bf16")
DTYPE = {"tf32": torch.float32, "bf16": torch.bfloat16}
E = {"tf32": 32, "bf16": 64}          # elements per 128-byte k-block row (K-major) / pixels per k-block (wgrad)
EXACT = 2 ** 24                       # integers below this are exact in fp32

# ---------------------------------------------------------------------------------------------------------------------
# Case tables.  inst = (mn, bn, pn): MN-major operands (weight gradient), tile width, column-piece width (0: none).
# ---------------------------------------------------------------------------------------------------------------------
Gemm = collections.namedtuple("Gemm", "id inst M N kb")
GEMM = [
    # N <= 64 -> BN 64.  300 rows: 3 tiles, the last one ragged (44 rows)
    Gemm("n48_kb1", (0, 64, 0), 300, 48, 1),               # one k-block
    Gemm("n48_stages", (0, 64, 0), 300, 48, 8),            # exactly the 8 ring stages
    # 8 + 1: ring wrap; 133 x 1 tiles on 132 CTAs; 48 % 32 != 0: no pieces
    Gemm("n48_wrap_133tiles", (0, 64, 0), 17000, 48, 9),
    # N = 200 -> BN 128, second column tile ragged (72 columns)
    Gemm("n200_kb1", (0, 128, 0), 1000, 200, 1),           # 8 x 2 tiles
    Gemm("n200_stages", (0, 128, 0), 1000, 200, 6),        # exactly the 6 ring stages
    Gemm("n200_wrap_142tiles", (0, 128, 0), 9000, 200, 7),  # ring wrap; 71 x 2 = 142 tiles: 2 units on 10 CTAs
    # N = 1024 -> BN 256 (N % 256 == 0)
    Gemm("n1024_kb1", (0, 256, 0), 129, 1024, 1),          # 2 x 4 tiles, second row tile holds one row
    Gemm("n1024_stages", (0, 256, 0), 1000, 1024, 4),      # exactly the 4 ring stages, 8 x 4 tiles
    # ring wrap; 50 x 4 = 200 tiles, last wave 68 > 66: whole tiles
    Gemm("n1024_wrap_200tiles", (0, 256, 0), 6350, 1024, 5),
    # column pieces of 64: 160 x 1 tiles, last wave 28 -> 4 pieces each (stage-3 conv2 of the step, K = 2304 in bf16)
    Gemm("conv2_pieces64", (0, 256, 64), 20480, 256, 36),
    # BN 256 because N > 1024; 30 x 5 = 150 tiles, last wave 18 -> 4 pieces; the last column tile holds 32 columns, so its
    # first piece is half beyond N and its other three pieces wholly beyond
    Gemm("n1056_pieces64", (0, 256, 64), 3840, 1056, 5),
    # column pieces of 128: 182 tiles, last wave 50 (50 x 4 > 132) -> 2 pieces each
    Gemm("m23296_pieces128", (0, 256, 128), 23296, 256, 10),
    Gemm("n512_pieces128", (0, 256, 128), 11648, 512, 10),  # 91 x 2 = 182 tiles, tail 50 -> 2 pieces
]

# Implicit-GEMM convolution, NHWC.  tile_w = the largest power of two <= 128 dividing Wo, tile_h = 128 / tile_w; the
# kernel's rows are M' = NB * tiles_per_img * 128 with tiles_per_img = Wo / tile_w * ceil(Ho / tile_h).
Conv = collections.namedtuple("Conv", "id inst NB H W Cin Cout k stride dil pad taps16 x_slice")
CONV = [
    Conv("tw128", (0, 64, 0), 1, 5, 128, 64, 64, 3, 1, 1, 1, False, False),      # Wo 128: tile 1 x 128, 5 tiles
    Conv("tw64_ho7", (0, 128, 0), 2, 7, 64, 128, 200, 3, 1, 1, 1, False, False),  # tile 2 x 64, Ho 7: 8 x 2 tiles
    Conv("tw32_ho10", (0, 256, 0), 2, 10, 32, 64, 1024, 3, 1, 1, 1, False, False),  # tile 4 x 32, Ho 10: 6 x 4 tiles
    Conv("tw16_ho13_1x1", (0, 64, 0), 2, 13, 48, 64, 48, 1, 1, 1, 0, False, False),  # Wo 48: tile 8 x 16, 3 x 2 per image
    # 16 explicit taps (kMaxTaps, a 4 x 4 window at offsets -1..2); Wo 24: tile 16 x 8, Ho 20: 3 x 2 per image
    Conv("tw8_ho20_16taps", (0, 128, 0), 1, 20, 24, 64, 96, 4, 1, 1, 1, True, False),
    Conv("stride2_ho31", (0, 128, 0), 2, 62, 64, 64, 128, 3, 2, 1, 1, False, False),  # Ho 31, Wo 32: tile 4 x 32, 16 tiles
    Conv("dil2_xslice", (0, 256, 0), 2, 16, 16, 128, 256, 3, 1, 2, 2, False, True),  # x a channel slice (x_ld > Cin)
    # 20 x 32 x 32 x 128 -> 256, 3 x 3: 20 x 8 = 160 tiles of 4 x 32 pixels, last wave 28 -> 4 pieces of 64 columns
    Conv("pieces64", (0, 256, 64), 20, 32, 32, 128, 256, 3, 1, 1, 1, False, False),
]

# model.Conv.bwd_data of a stride-2 layer: k = 1 writes every other pixel through out_map; k = 3 runs four parity-class
# convolutions over dY (1, 2, 2 and 4 taps of the transposed weights).  Each is a conv over the H/2 x W/2 grid with
# N = cin: 2 images of 32 x 32 -> tile 4 x 32, 16 tiles per column tile.
Dgrad = collections.namedtuple("Dgrad", "id inst NB H W cin cout k")
DGRAD = [
    Dgrad("k1_s2", (0, 256, 0), 2, 64, 64, 256, 64, 1),
    Dgrad("k3_s2", (0, 128, 0), 2, 64, 64, 128, 64, 3),
]

# Weight gradient dW[Cout, taps * Cin] (mode 2, MN-major operands).  BN = 256 / 128 / 64 for Cin % 256 / % 128 / else;
# k-blocks are kp = 32 (tf32) / 64 (bf16) consecutive output pixels; tiles = ceil(Cout / 128) * taps * Cin / BN.  Cout
# (None) = 96 for tf32 (one ragged row tile) and 192 for bf16 (128 + 64).  Requested splits are cut to the largest
# s <= splits with total_kb % s == 0 and tiles * s <= 132; 0 = auto (fill one wave, at least 8 k-blocks per split).
Wgrad = collections.namedtuple("Wgrad", "id inst NB H W Cin Cout k stride dil pad splits slices accumulate")
WGRAD = [
    # Wo 16 < kp (tf32 2, bf16 4 image rows per k-block).  512 px: 16 / 8 k-blocks; tiles 9 / 18
    Wgrad("bn64_wo16", (1, 64, 0), 2, 16, 16, 64, None, 3, 1, 1, 1, 1, False, False),
    # Wo 8 < kp (tf32 4, bf16 8 rows per k-block).  128 px: 4 / 2 k-blocks, 2 splits; tiles 9 / 18
    Wgrad("bn128_wo8_split2", (1, 128, 0), 2, 8, 8, 128, None, 3, 1, 1, 1, 2, False, False),
    # bf16 Wo 32 < kp.  2048 px: 64 / 32 k-blocks, neither divisible by 3: 3 splits are cut to 2; tiles 9 / 18
    Wgrad("bn256_wo32_split3", (1, 256, 0), 2, 32, 32, 256, None, 3, 1, 1, 1, 3, False, False),
    # stride 2, 9 taps, Cin 512 (2 column blocks per tap): tiles 18 / 36; 8 splits need 144 / 288 > 132 units:
    # tf32 7, 6, 5 do not divide 64 k-blocks -> 4; bf16 <= 3 by the unit cap, 3 does not divide 32 -> 2
    Wgrad("bn256_stride2_split8", (1, 256, 0), 2, 64, 64, 512, None, 3, 2, 1, 1, 8, False, False),
    # dilation 2, 9 taps, auto splits: tf32 tiles 9 -> (132 + 4) / 9 = 15, capped at 64 / 8 = 8; bf16 tiles 18 -> 7,
    # capped at 32 / 8 = 4
    Wgrad("bn128_dil2_auto", (1, 128, 0), 2, 32, 32, 128, None, 3, 1, 2, 2, 0, False, False),
    # dY and X channel slices (dy_ld > Cout, x_ld > Cin), accumulated onto a non-zero dW; 1 x 1, 8 splits of
    # 64 / 32 k-blocks, tiles 1 / 2
    Wgrad("bn64_slices_accumulate", (1, 64, 0), 2, 32, 32, 64, None, 1, 1, 1, 0, 8, True, True),
    # fc_new_1 of the step: dY [1,1,6000,1024], X [1,1,6000,12544] (a single pixel row).  8 x 49 = 392 tiles: 2-3 units per
    # CTA, so the TMA ring (and the tf32 transpose ring) carry their phase across units; 6000 % kp != 0: the TMA
    # zero-fills the last k-block (188 / 94 k-blocks); auto splits stay at 1 (392 >= 132 tiles)
    Wgrad("fc_new_1", (1, 256, 0), 1, 1, 6000, 12544, 1024, 1, 1, 1, 0, 0, False, False),
]


def conv_out_hw(c):
    if c.taps16:
        return c.H, c.W
    Ho = (c.H + 2 * c.pad - c.dil * (c.k - 1) - 1) // c.stride + 1
    Wo = (c.W + 2 * c.pad - c.dil * (c.k - 1) - 1) // c.stride + 1
    return Ho, Wo


def conv_tile(Wo):
    """(tile_h, tile_w) of sniper_conv2d_nhwc for an output width Wo"""
    tw = 128
    while Wo % tw:
        tw //= 2
    return 128 // tw, tw


def conv_rows(NB, Ho, Wo):
    """M' = the kernel's row count for an NB x Ho x Wo output: NB * tiles_per_img * 128"""
    th, tw = conv_tile(Wo)
    return NB * (Wo // tw) * (-(-Ho // th)) * 128


def wgrad_cout(w, dt):
    return w.Cout if w.Cout is not None else (96 if dt == "tf32" else 192)


def wgrad_tiles(w, dt):
    bn = w.inst[1]
    return -(-wgrad_cout(w, dt) // 128) * w.k * w.k * (w.Cin // bn)


# ---------------------------------------------------------------------------------------------------------------------
# exact comparison helpers
# ---------------------------------------------------------------------------------------------------------------------
def _gen(seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return g


def _ints(g, shape, lo, hi, dtype=torch.float32):
    return torch.randint(lo, hi + 1, tuple(shape), device="cuda", generator=g).to(dtype)


def _check_range(ref):
    """Exactness precondition: every value of the exact result below 2^24"""
    m = ref.abs().max().item() if ref.numel() else 0.0
    assert m < EXACT, "case is not exact in fp32: max |value| %g >= 2^24 (change the case)" % m


def _same(got, ref, dtype, what=""):
    """got (any shape, any strides) == ref (float64 [R, N]) rounded to dtype (RNE for bf16), bit for bit."""
    _check_range(ref)
    exp = ref.to(dtype)
    got = got.reshape(exp.shape)
    if torch.equal(got, exp):
        return
    d = got.double() - exp.double()
    bad = d.ne(0).nonzero()
    rows, cols = bad[:, 0], bad[:, 1]
    first = ", ".join("(%d,%d): %+g" % (int(r), int(c), float(d[r, c])) for r, c in bad[:8].tolist())
    raise AssertionError("%s: %d of %d values differ; rows %d..%d, columns %d..%d; first: %s" % (
        what, bad.shape[0], d.numel(), int(rows.min()), int(rows.max()), int(cols.min()), int(cols.max()), first))


def _same_stats(st, y, tile, what=""):
    """Fused statistics == column sums / sums of squares of the stored values y (float64 [R, N]).  Precondition: every
    128-row tile's per-column sum of squares < 2^24 (the kernel sums a tile in fp32; squares are >= |value|)."""
    N = y.shape[1]
    sq = torch.zeros(int(tile.max()) + 1, N, dtype=torch.float64, device=y.device).index_add_(0, tile, y * y)
    assert sq.max().item() < EXACT, "case is not exact: a tile's sum of squares is %g >= 2^24" % sq.max().item()
    ref = torch.cat([y.sum(0), (y * y).sum(0)])
    if not torch.equal(st, ref):
        d = (st - ref).ne(0).nonzero().flatten().tolist()
        raise AssertionError("%s statistics: %d of %d differ, first entries %s" % (what, len(d), 2 * N, d[:8]))


def _check_epilogues(run, acc, tile, out_shape, dt, g, what):
    """run(**epilogue) launches the op (gemm_nt / conv2d_nhwc keywords); acc = the exact float64 accumulator as [R, N] in
    output row order; tile[r] = the kernel tile that stores row r."""
    _check_range(acc)
    R, N = acc.shape
    odt = DTYPE[dt]
    other = torch.bfloat16 if odt == torch.float32 else torch.float32
    scale = 2.0 ** _ints(g, (N,), 0, 1)
    bias = _ints(g, (N,), -4, 4)
    sc, bi = scale.double(), bias.double()
    # plain store
    _same(run(), acc, odt, what + " plain")
    # scale + bias + relu, fused statistics of the stored values
    st = torch.zeros(2 * N, dtype=torch.float64, device="cuda")
    ref = (acc * sc + bi).clamp_min(0)
    _same(run(scale=scale, bias=bias, relu=True, stats=st), ref, odt, what + " scale/bias/relu")
    _same_stats(st, ref.to(odt).double(), tile, what)
    # residual in place (out is residual)
    o = _ints(g, out_shape, -4, 4, odt)
    ref = acc + o.reshape(R, N).double()
    run(out=o, residual=o)
    _same(o, ref, odt, what + " residual in place")
    # accumulate into an fp32 output
    o = _ints(g, out_shape, -8, 8)
    ref = acc + bi + o.reshape(R, N).double()
    run(out=o, bias=bias, accumulate=True)
    _same(o, ref, torch.float32, what + " accumulate")
    # column slices of wider buffers (ld > N), as the concat buffers use them; the other columns stay untouched
    big = torch.full(tuple(out_shape[:-1]) + (N + 64,), 7.0, dtype=odt, device="cuda")
    rbig = _ints(g, tuple(out_shape[:-1]) + (N + 32,), -4, 4, odt)
    res = rbig[..., 16:16 + N]
    run(out=big[..., 32:32 + N], residual=res, bias=bias)
    _same(big[..., 32:32 + N], acc + bi + res.reshape(R, N).double(), odt, what + " column slices")
    assert bool((big[..., :32] == 7).all()) and bool((big[..., 32 + N:] == 7).all()), what + ": store outside the slice"
    # the other output type (tf32 operands -> bf16 output, bf16 operands -> fp32 output) with its residual and statistics
    r = _ints(g, out_shape, -4, 4, other)
    st = torch.zeros(2 * N, dtype=torch.float64, device="cuda")
    ref = (acc * sc + bi + r.reshape(R, N).double()).clamp_min(0)
    out = run(out_dtype=other, residual=r, scale=scale, bias=bias, relu=True, stats=st)
    assert out.dtype == other
    _same(out, ref, other, what + " output type")
    _same_stats(st, ref.to(other).double(), tile, what + " output type")


def _operands(g, dt, *shapes):
    return [_ints(g, s, -1, 1, DTYPE[dt]) for s in shapes]


# ---------------------------------------------------------------------------------------------------------------------
# K-major GEMM
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", GEMM, ids=lambda c: c.id)
def test_gemm_exact(case, dt):
    from sniper_b200 import ops
    g = _gen(case.M + case.N + case.kb)
    K = case.kb * E[dt]
    a, b = _operands(g, dt, (case.M, K), (case.N, K))
    acc = a.double() @ b.double().t()
    tile = torch.arange(case.M, device="cuda") // 128
    _check_epilogues(lambda **kw: ops.gemm_nt(a, b, **kw), acc, tile, (case.M, case.N), dt, g,
                     "%s %s" % (case.id, dt))


# ---------------------------------------------------------------------------------------------------------------------
# implicit-GEMM convolution
# ---------------------------------------------------------------------------------------------------------------------
def _conv_tile_index(NB, Ho, Wo):
    th, tw = conv_tile(Wo)
    n = torch.arange(NB, device="cuda").view(-1, 1, 1)
    oh = torch.arange(Ho, device="cuda").view(1, -1, 1)
    ow = torch.arange(Wo, device="cuda").view(1, 1, -1)
    per_img = (Wo // tw) * (-(-Ho // th))
    return (n * per_img + (oh // th) * (Wo // tw) + ow // tw).flatten()


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", CONV, ids=lambda c: c.id)
def test_conv_exact(case, dt):
    import torch.nn.functional as F
    from sniper_b200 import ops
    c = case
    g = _gen(c.H * 7 + c.Cin + c.Cout + c.k)
    Ho, Wo = conv_out_hw(c)
    if c.x_slice:
        xbig, w = _operands(g, dt, (c.NB, c.H, c.W, c.Cin + 64), (c.Cout, c.k, c.k, c.Cin))
        x = xbig[..., 32:32 + c.Cin]
    else:
        x, w = _operands(g, dt, (c.NB, c.H, c.W, c.Cin), (c.Cout, c.k, c.k, c.Cin))
    xd, wd = x.double().permute(0, 3, 1, 2), w.double().permute(0, 3, 1, 2)
    if c.taps16:
        # taps at offsets -1..2 in both directions: pad 1 before, 2 after, then a plain 4 x 4 correlation
        taps = ops.conv_taps(4, 4, 1, 1)
        assert len(taps[0]) == 16 and min(taps[0]) == -1 and max(taps[0]) == 2
        ref = F.conv2d(F.pad(xd, (1, 2, 1, 2)), wd)
        kw = dict(kh=0, kw=0, taps=taps, out_hw=(Ho, Wo))
    else:
        ref = F.conv2d(xd, wd, stride=c.stride, padding=c.pad, dilation=c.dil)
        kw = dict(kh=c.k, kw=c.k, stride=c.stride, dil=c.dil, pad=c.pad)
    assert ref.shape[2:] == (Ho, Wo)
    acc = ref.permute(0, 2, 3, 1).reshape(-1, c.Cout)
    wr = w.reshape(c.Cout, -1).contiguous()
    _check_epilogues(lambda **e: ops.conv2d_nhwc(x, wr, **kw, **e), acc, _conv_tile_index(c.NB, Ho, Wo),
                     (c.NB, Ho, Wo, c.Cout), dt, g, "%s %s" % (c.id, dt))


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", DGRAD, ids=lambda c: c.id)
def test_conv_bwd_data_stride2_exact(case, dt):
    """model.Conv.bwd_data of a stride-2 layer: the weight transpose and the out_map phase writes, against autograd."""
    import torch.nn.functional as F
    from sniper_b200 import model
    c = case
    g = _gen(c.H + c.cin + c.k)
    lowp = dt == "bf16"
    P = model.ParamStore()
    conv = model.Conv(P, "c", c.cin, c.cout, k=c.k, stride=2, pad=c.k // 2, lowp=lowp)
    P.finalize("cuda", lowp=lowp)
    w = _ints(g, (c.cout, c.k, c.k, c.cin), -1, 1)
    P["c_weight"].copy_(w.reshape(c.cout, -1))
    P.sync_lowp()
    conv.prepare_bwd()
    Ho, Wo = c.H // 2, c.W // 2
    dy = _ints(g, (c.NB, Ho, Wo, c.cout), -1, 1, DTYPE[dt])
    dx = conv.bwd_data(dy, (c.H, c.W))
    xd = torch.zeros(c.NB, c.cin, c.H, c.W, dtype=torch.float64, device="cuda", requires_grad=True)
    F.conv2d(xd, w.double().permute(0, 3, 1, 2), stride=2, padding=c.k // 2).backward(dy.double().permute(0, 3, 1, 2))
    ref = xd.grad.permute(0, 2, 3, 1).reshape(-1, c.cin)
    assert dx.shape == (c.NB, c.H, c.W, c.cin)
    _same(dx, ref, DTYPE[dt], "%s %s" % (c.id, dt))


def test_accumulate_into_bf16_output_is_refused():
    """The epilogue stores bf16 outputs and never adds to them, so accumulate=True with a bf16 output is an error."""
    from sniper_b200 import ops
    from sniper_b200._lib import SniperError
    a = torch.ones(128, 64, device="cuda", dtype=torch.bfloat16)
    c = torch.ones(128, 128, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(SniperError, match="accumulate"):
        ops.gemm_nt(a, a, out=c, accumulate=True)
    with pytest.raises(SniperError, match="accumulate"):
        ops.gemm_nt(a.float(), a.float(), out=c, accumulate=True)
    x = torch.ones(1, 8, 16, 64, device="cuda", dtype=torch.bfloat16)
    y = torch.ones(1, 8, 16, 128, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(SniperError, match="accumulate"):
        ops.conv2d_nhwc(x, a, kh=1, kw=1, out=y, accumulate=True)
    torch.cuda.synchronize()
    assert bool((c == 1).all()) and bool((y == 1).all())


# ---------------------------------------------------------------------------------------------------------------------
# weight gradients
# ---------------------------------------------------------------------------------------------------------------------
def _wgrad_ref(dy, x, k, stride, dil, pad):
    """float64 dW [Cout, k*k*Cin] (tap-major, channel-minor) of F.conv2d by autograd; dy / x NHWC"""
    import torch.nn.functional as F
    Cout, Cin = dy.shape[3], x.shape[3]
    if k == 1 and stride == 1 and pad == 0:
        return dy.double().reshape(-1, Cout).t() @ x.double().reshape(-1, Cin)
    wd = torch.zeros(Cout, Cin, k, k, dtype=torch.float64, device="cuda", requires_grad=True)
    F.conv2d(x.double().permute(0, 3, 1, 2), wd, stride=stride, padding=pad, dilation=dil).backward(
        dy.double().permute(0, 3, 1, 2))
    return wd.grad.permute(0, 2, 3, 1).reshape(Cout, -1)


def _wgrad_inputs(w, dt, g):
    Cout = wgrad_cout(w, dt)
    Ho = (w.H + 2 * w.pad - w.dil * (w.k - 1) - 1) // w.stride + 1
    Wo = (w.W + 2 * w.pad - w.dil * (w.k - 1) - 1) // w.stride + 1
    if w.slices:
        dyb, xb = _operands(g, dt, (w.NB, Ho, Wo, Cout + 64), (w.NB, w.H, w.W, w.Cin + 64))
        return dyb[..., 32:32 + Cout], xb[..., 64:64 + w.Cin]
    return _operands(g, dt, (w.NB, Ho, Wo, Cout), (w.NB, w.H, w.W, w.Cin))


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", WGRAD, ids=lambda c: c.id)
def test_wgrad_exact(case, dt):
    from sniper_b200 import ops
    w = case
    g = _gen(w.H + w.Cin + w.k + w.splits)
    dy, x = _wgrad_inputs(w, dt, g)
    ref = _wgrad_ref(dy, x, w.k, w.stride, w.dil, w.pad)
    dw = _ints(g, ref.shape, -8, 8) if w.accumulate else torch.zeros(ref.shape, device="cuda")
    if w.accumulate:
        ref = ref + dw.double()
    ops.conv2d_wgrad_nhwc(dy, x, kh=w.k, kw=w.k, stride=w.stride, dil=w.dil, pad=w.pad, dw_out=dw, splits=w.splits)
    _same(dw, ref, torch.float32, "%s %s" % (w.id, dt))


def test_bias_gradient_colsum_exact():
    """ops.colsum_accum (the bias gradient next to each weight gradient): C not a multiple of 32, M not a multiple of 128,
    a channel slice (ld > C), accumulated onto non-zero values."""
    from sniper_b200 import ops
    g = _gen(11)
    for M, C in [(6000, 85), (20000, 1000), (97, 33)]:
        big = _ints(g, (M, C + 40), -3, 3)
        x = big[:, 8:8 + C]
        out = _ints(g, (C,), -100, 100)
        ref = out.double() + x.double().sum(0)
        ops.colsum_accum(x, out)
        _same(out.view(1, C), ref.view(1, C), torch.float32, "colsum %dx%d" % (M, C))


# ---------------------------------------------------------------------------------------------------------------------
# split-K through the stream's workspace: on any number of streams, at once, and under graph replay
# ---------------------------------------------------------------------------------------------------------------------
def _split_k_problem(dt, seed):
    """1 x 1 weight gradient over 4 x 32 x 32 pixels, Cin 256: 128 / 64 k-blocks, tiles 1 / 2, 8 splits either way"""
    w = Wgrad("split8", (1, 256, 0), 4, 32, 32, 256, None, 1, 1, 1, 0, 8, False, False)
    dy, x = _wgrad_inputs(w, dt, _gen(seed))
    return dy, x, _wgrad_ref(dy, x, 1, 1, 1, 0)


# The stream's workspace (ops._stream_workspace) starts with the split-K regions: [parked partials: 132 x 128 x 256 fp32 |
# arrival counters: 132 x 8 int32].
PARKED_BYTES, COUNTER_BYTES = 132 * 128 * 256 * 4, 132 * 8 * 4
POISON = -12345.0       # no parked partial of _split_k_problem can take this value (|partial| <= 4096 pixels)


def _split_k_views(stream):
    """(parked partials, arrival counters) of the stream's workspace"""
    from sniper_b200 import ops
    with torch.cuda.stream(stream):
        ws = ops._stream_workspace()
    return ws[:PARKED_BYTES].view(torch.float32), ws[PARKED_BYTES:PARKED_BYTES + COUNTER_BYTES].view(torch.int32)


def _poison(streams):
    torch.cuda.synchronize()
    for s in streams:
        parked, _ = _split_k_views(s)
        with torch.cuda.stream(s):          # after the zero fill of a workspace created just now
            parked.fill_(POISON)
    torch.cuda.synchronize()


def _split_k_ran(stream):
    """whether a launch on the stream wrote its parked-partials region since the last _poison (i.e. ran a split-K
    reduction), with every arrival counter back at zero"""
    torch.cuda.synchronize()
    parked, cnt = _split_k_views(stream)
    assert not bool(cnt.any()), "split-K counters were left non-zero"
    return bool((parked != POISON).any())


def _split_k_on_streams(dt, streams, seed):
    """One split-K weight gradient per stream, all held behind one event so that they run at the same time; each exact"""
    from sniper_b200 import ops
    probs = [_split_k_problem(dt, seed + i) for i in range(len(streams))]
    main = torch.cuda.current_stream()
    gate = torch.cuda.Event()
    torch.cuda._sleep(20_000_000)            # ~10 ms: every launch below is queued before the gate opens
    gate.record(main)
    outs = []
    for s, (dy, x, _) in zip(streams, probs):
        s.wait_event(gate)
        with torch.cuda.stream(s):
            dw = torch.zeros(dy.shape[3], x.shape[3], device="cuda")
            ops.conv2d_wgrad_nhwc(dy, x, kh=1, kw=1, dw_out=dw, splits=8)
            outs.append(dw)
    torch.cuda.synchronize()
    for i, (dw, (_, _, ref)) in enumerate(zip(outs, probs)):
        _same(dw, ref, torch.float32, "stream %d of %d (%s)" % (i, len(streams), dt))


@pytest.mark.parametrize("dt", DTS)
def test_split_k_on_concurrent_streams(dt):
    """Split-K weight gradients on seven streams at once each run split in their own stream's workspace and are each
    exact."""
    streams = [torch.cuda.Stream() for _ in range(7)]
    assert len({s.cuda_stream for s in streams} | {torch.cuda.current_stream().cuda_stream}) == 8
    _poison(streams)
    _split_k_on_streams(dt, streams, 100)
    assert [_split_k_ran(s) for s in streams] == [True] * 7, "not every stream ran split-K"


def test_split_k_is_byte_equal_on_every_stream():
    """The split count depends on the shape alone: the same 8-split weight gradient on random fp32 operands gives the
    same bytes on six fresh streams, and each of them runs the split-K reduction, however many streams this process
    has used before."""
    from sniper_b200 import ops
    g = _gen(400)
    dy = torch.randn(4, 32, 32, 96, device="cuda", generator=g)
    x = torch.randn(4, 32, 32, 256, device="cuda", generator=g)
    streams = [torch.cuda.Stream() for _ in range(6)]
    assert len({s.cuda_stream for s in streams}) == 6
    _poison(streams)
    outs = []
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            outs.append(ops.conv2d_wgrad_nhwc(dy, x, kh=1, kw=1, splits=8))
    torch.cuda.synchronize()
    for i, dw in enumerate(outs):
        assert torch.equal(dw.view(torch.int32), outs[0].view(torch.int32)), "stream %d differs from stream 0" % i
    assert [_split_k_ran(s) for s in streams] == [True] * 6, "not every stream ran split-K"


@pytest.mark.parametrize("dt", DTS)
def test_split_k_on_an_unregistered_stream_is_refused(dt):
    """A split-K launch needs its stream's workspace: on a fabricated stream handle nothing was registered for, the
    call is refused before any launch and dW stays untouched."""
    import ctypes
    from sniper_b200._lib import lib
    dy, x, ref = _split_k_problem(dt, 500)
    dw = torch.zeros(ref.shape, device="cuda")
    NB, H, W, Cin = x.shape
    Cout = dy.shape[3]
    zero = ctypes.c_int(0)
    L = lib()
    rc = L.sniper_conv2d_wgrad_nhwc(dy.data_ptr(), Cout, x.data_ptr(), Cin, NB, H, W, Cin, Cout, 1,
                                    ctypes.addressof(zero), ctypes.addressof(zero), 1, H, W, dw.data_ptr(),
                                    0 if dt == "tf32" else 1, 8, 0x7f00beef2000)
    err = L.sniper_last_error().decode()
    assert rc != 0 and "wgrad: no workspace registered for this stream (sniper_set_stream_workspace)" in err, err
    torch.cuda.synchronize()
    assert not bool(dw.any())


def test_graph_replay_column_pieces_and_split_k():
    """One CUDA graph holding a column-piece GEMM and a split-K weight gradient, captured on a stream and replayed
    twice: each replay runs the split-K reduction (it writes the capture stream's parked partials), equals the exact
    results, and leaves every arrival counter at zero."""
    from sniper_b200 import ops
    g = _gen(300)
    M, N, K = 20480, 256, 4 * 32            # 160 tiles, last wave 28 -> 64-column pieces
    a, b = _operands(g, "tf32", (M, K), (N, K))
    ref_c = a.double() @ b.double().t()
    dy, x, ref_w = _split_k_problem("tf32", 301)
    c = torch.zeros(M, N, device="cuda")
    dw = torch.zeros(ref_w.shape, device="cuda")
    cs = torch.cuda.Stream()
    _poison([cs])
    cs.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(cs):             # eager on the capture stream first
        ops.gemm_nt(a, b, out=c)
        ops.conv2d_wgrad_nhwc(dy, x, kh=1, kw=1, dw_out=dw, splits=8)
    torch.cuda.synchronize()
    _same(c, ref_c, torch.float32, "eager gemm")
    _same(dw, ref_w, torch.float32, "eager wgrad")
    assert _split_k_ran(cs)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=cs):
        dw.zero_()
        ops.gemm_nt(a, b, out=c)
        ops.conv2d_wgrad_nhwc(dy, x, kh=1, kw=1, dw_out=dw, splits=8)
    for i in range(2):
        c.fill_(-5.0)
        dw.fill_(-5.0)
        _poison([cs])
        graph.replay()
        torch.cuda.synchronize()
        _same(c, ref_c, torch.float32, "replay %d gemm" % i)
        _same(dw, ref_w, torch.float32, "replay %d wgrad" % i)
        assert _split_k_ran(cs), "replay %d did not run the split-K reduction" % i


# ---------------------------------------------------------------------------------------------------------------------
# operand rounding, per operand path, on random data
# ---------------------------------------------------------------------------------------------------------------------
def _tf32_trunc(x):
    return (x.float().contiguous().view(torch.int32) & -8192).view(torch.float32).double()


def _tf32_rne(x):
    i = x.float().contiguous().view(torch.int32)
    i = i + 0x0FFF + ((i >> 13) & 1)
    return (i & -8192).view(torch.float32).double()


def _rel(a, b):
    return ((a.double() - b).norm() / b.norm()).item()


def _conv_randn(dtype):
    """3 x 3 conv, 2 x 32 x 32 x 128 -> 256: returns (x, w, y, ref(xd, wd)) with y from the kernel"""
    import torch.nn.functional as F
    from sniper_b200 import ops
    torch.manual_seed(21)
    x = torch.randn(2, 32, 32, 128, device="cuda").to(dtype)
    w = torch.randn(256, 3, 3, 128, device="cuda").to(dtype)
    y = ops.conv2d_nhwc(x, w.reshape(256, -1).contiguous(), kh=3, kw=3, pad=1, out_dtype=torch.float32)

    def ref(xd, wd):
        return F.conv2d(xd.permute(0, 3, 1, 2), wd.permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1)
    return x, w, y, ref


def _wgrad_randn(dtype):
    """3 x 3 weight gradient, 1 x 32 x 32 pixels, Cin 128, Cout 192, 4 splits"""
    from sniper_b200 import ops
    torch.manual_seed(22)
    x = torch.randn(1, 32, 32, 128, device="cuda").to(dtype)
    dy = torch.randn(1, 32, 32, 192, device="cuda").to(dtype)
    dw = ops.conv2d_wgrad_nhwc(dy, x, kh=3, kw=3, pad=1, splits=4)
    return x, dy, dw, lambda xd, dyd: _wgrad_ref(dyd, xd, 3, 1, 1, 1)


@pytest.mark.parametrize("path", ["conv", "wgrad"])
def test_tf32_operands_truncate(path):
    """TF32 reads ignore the low 13 mantissa bits of each fp32 word: the conv (4-D TMA operand) and the weight gradient
    (MN-major operands transposed by the consumers) equal float64 on TRUNCATED operands to accumulation noise and sit
    far from round-to-nearest operands.  A transpose that converted (cvt.rna) instead of copying words would flip this."""
    p, q, y, ref = (_conv_randn if path == "conv" else _wgrad_randn)(torch.float32)
    torch.cuda.synchronize()
    et, er = _rel(y, ref(_tf32_trunc(p), _tf32_trunc(q))), _rel(y, ref(_tf32_rne(p), _tf32_rne(q)))
    print("%s: vs truncated operands %.2e, vs RNE operands %.2e" % (path, et, er))
    assert et < 5e-6 and er > 20 * et


@pytest.mark.parametrize("path", ["gemm", "conv", "wgrad"])
def test_bf16_operands_exact_products(path):
    """bf16 operands are exact: every operand path equals float64 on the bf16 values to fp32 accumulation noise."""
    from sniper_b200 import ops
    if path == "gemm":
        torch.manual_seed(23)
        p = torch.randn(512, 1024, device="cuda").bfloat16()
        q = torch.randn(256, 1024, device="cuda").bfloat16()
        y = ops.gemm_nt(p, q, out_dtype=torch.float32)

        def ref(a, b):
            return a @ b.t()
    else:
        p, q, y, ref = (_conv_randn if path == "conv" else _wgrad_randn)(torch.bfloat16)
    torch.cuda.synchronize()
    e = _rel(y, ref(p.double(), q.double()))
    print("%s: bf16 vs float64 %.2e" % (path, e))
    assert e < 5e-6


# ---------------------------------------------------------------------------------------------------------------------
# input checks of the wrappers (all fail on the host, before any launch)
# ---------------------------------------------------------------------------------------------------------------------
def test_wrappers_refuse_bad_operands():
    from sniper_b200 import ops
    a = torch.zeros(256, 64, device="cuda")
    b = torch.zeros(128, 64, device="cuda")
    with pytest.raises(AssertionError):
        ops.gemm_nt(a, b, out=torch.zeros(256, 64, device="cuda"))                     # out not [M, N]
    with pytest.raises(AssertionError):
        ops.gemm_nt(a, b, out=torch.zeros(128, 256, device="cuda").t())                # out column stride != 1
    with pytest.raises(AssertionError):
        ops.gemm_nt(a, b, residual=torch.zeros(256, 64, device="cuda"))                # residual not [M, N]
    with pytest.raises(AssertionError):
        ops.gemm_nt(a, b, residual=torch.zeros(128, 256, device="cuda").t())           # residual column stride != 1
    dy = torch.zeros(2, 8, 8, 64, device="cuda")
    x = torch.zeros(2, 8, 8, 64, device="cuda")
    with pytest.raises(AssertionError):
        ops.conv2d_wgrad_nhwc(dy[:, :, :4], x[:, :, :4], kh=1, kw=1)                   # rows not uniformly strided
    with pytest.raises(AssertionError):
        ops.conv2d_wgrad_nhwc(dy, x.permute(0, 2, 1, 3), kh=1, kw=1)                   # x rows not uniformly strided
    with pytest.raises(AssertionError):
        ops.conv2d_wgrad_nhwc(dy, x, kh=1, kw=1, dw_out=torch.zeros(64, 64, device="cuda", dtype=torch.float64))
    with pytest.raises(AssertionError):
        ops.conv2d_wgrad_nhwc(dy, x, kh=1, kw=1, dw_out=torch.zeros(64, 128, device="cuda")[:, :64])  # not contiguous
    with pytest.raises(AssertionError):
        ops.conv2d_wgrad_nhwc(dy, x, kh=3, kw=3, pad=1, dw_out=torch.zeros(64, 64, device="cuda"))  # not [Cout, 9 Cin]
    with pytest.raises(AssertionError):
        ops.colsum_accum(torch.zeros(100, 64, device="cuda", dtype=torch.bfloat16), torch.zeros(64, device="cuda"))
