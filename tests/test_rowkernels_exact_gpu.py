"""BatchNorm / elementwise row kernels (csrc/elementwise.cu, add_rows of csrc/depthwise.cu) against float64, at every
geometry `row_block()` can choose.

Each case runs a public `sniper_b200.ops` wrapper and compares with a plain float64 PyTorch evaluation of the same
operation ON THE STORED INPUTS (the bf16-rounded tensor for bf16 storage).  One seeded generator per case, so a failing
id (dtype-M-C) names its shape.

Shape grid.  C in C_F32 / C_BF16 covers lx_shift 3 / 4 / 5 (C / vec < 16, < 32, >= 32 with vec = 4 fp32 / 8 bf16),
rows narrower than one slab (C / vec < LX), full and ragged last slabs (bf16 144, 576, 960, 1280, ...), and power-of-two
and other C / 4 (RowSplit's two paths).  M covers fewer rows than one thread row (RY = 8 / 16 / 32), RY - 1 / RY / RY + 1,
one row either side of four unrolled trips (4 * RY * KU -+ 1), and the two mid sizes the older tests used.  The cross
product is pruned to: every C at M = 4 * RY * KU + 1 and M = 5000; every M at C = 24, 144 and 1024; strided / in-place
layouts at the LAYOUTS shapes; and once per dtype the real stem shape, 20 chips x 256 x 256 = 1 310 720 rows of 64
channels (statistics, fused apply and backward only; its float64 reference is built in chunks).

Bounds.  Pointwise results: 1 ulp of the storage type (fp32: 2^-23 |ref| + one denormal; bf16: half a bf16 ulp with 1 %
slack for the double rounding through fp32 + 1e-6), bit-equality where the operation is exact.  Sums: the kernels add at
most n_t <= sqrt(M) + 4 terms per thread in fp32 (n_t = rows a thread walks: one wave of >= 2 blocks per SM over 132 SMs
leaves n_t <= 16 M / (248 RY); at the stem shape n_t ~ 150 against sqrt(M) = 1145) and everything above a thread in
double, so |error| <= K(M) * sum|terms| with K(M) = (4 + sqrt(M)) * 2^-24 is a worst-case bound, not a statistical one.
Mask elements whose float64 pre-activation lies within the rounding of the kernel's own fma of a clip boundary may take
either side: they are counted (must stay below 1e-4 of the tensor), excluded from the per-element comparison, and their
gradient is added to the tolerance of the sums they feed.

`test_zz_report` prints the worst error seen per assertion class next to its bound (run with -s).  Measured on an H100
80GB HBM3 (700 W): pointwise kernels 0.50 ulp fp32 / 0.99 of the bf16 bound; relative variance error of bn_stats with
|mean| = 100 std: 5.0e-4 worst over the grid and 6.5e-5 at the stem shape in fp32 storage (1e-7 in bf16 storage, whose
few distinct values sum exactly), against the enforced 1e-3; with mean 0.5 / std 2 it is 1.5e-7; dx of the backward
within 0.88 of its bound in fp32; run-to-run results bit-identical everywhere."""
import math

import pytest

pytestmark = pytest.mark.gpu

DEV = "cuda"
KU = 4                       # unrolled loads per operand per thread (VT<T>::U)
E32 = 2.0 ** -23             # one fp32 ulp, relative
BF = 2.0 ** -8               # half a bf16 ulp, relative
EPS = 2e-5
CHUNK = 1 << 17              # rows of float64 reference held at a time

C_F32 = [4, 8, 12, 16, 20, 24, 32, 64, 96, 144, 192, 256, 320, 576, 960, 1024, 1280, 2048]
C_BF16 = [c for c in C_F32 if c % 8 == 0]
STEM = (20 * 256 * 256, 64)

WORST = {}                   # assertion class -> (worst error / bound, worst error, its bound)


def _note(what, err, bound):
    import torch
    ratio = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, float("inf"), 0.0).double())
    i = int(ratio.reshape(-1).argmax())
    r = (float(ratio.reshape(-1)[i]), float(err.reshape(-1)[i]), float(bound.reshape(-1)[i]))
    if what not in WORST or r[0] > WORST[what][0]:
        WORST[what] = r


def _within(what, got, ref, bound, skip=None):
    """|got - ref| <= bound everywhere (except `skip`), no NaN / Inf; records the worst ratio."""
    import torch
    got = got.double()
    assert bool(torch.isfinite(got).all()), what + ": NaN / Inf in the result"
    err = (got - ref).abs()
    if skip is not None:
        err = err * (~skip)
    bound = torch.broadcast_to(bound, err.shape)
    _note(what, err, bound)
    bad = err > bound
    assert not bool(bad.any()), "%s: %d elements out of bound, worst excess %.3e" % (
        what, int(bad.sum()), float((err - bound).max()))


def _ulp_bound(ref, dtype):
    import torch
    if dtype == torch.float32:
        return ref.abs() * E32 + 2.0 ** -149
    return ref.abs() * BF * 1.01 + 1e-6


def _dt(name):
    import torch
    return getattr(torch, name)


def _vecw(dt):
    return 4 if dt == "float32" else 8


def _ry(C, dt):
    cv = C // _vecw(dt)
    return 8 if cv >= 32 else (16 if cv >= 16 else 32)


def _m_values(C, dt):
    ry = _ry(C, dt)
    return [1, 7, ry - 1, ry, ry + 1, 4 * ry * KU - 1, 4 * ry * KU + 1, 5000, 20504]


def _grid():
    cases = []
    for dt in ("float32", "bfloat16"):
        for C in (C_F32 if dt == "float32" else C_BF16):
            for M in (4 * _ry(C, dt) * KU + 1, 5000):
                cases.append((dt, M, C))
        for C in (24, 144, 1024):
            for M in _m_values(C, dt):
                if (dt, M, C) not in cases:
                    cases.append((dt, M, C))
    return cases


GRID = _grid()
# a quarter of the grid (every 4th case + all the C = 24 / 144 cases with few rows) for the tests that loop over flags
SMALL = [c for i, c in enumerate(GRID) if i % 4 == 0 or (c[2] in (24, 144) and c[1] < 40)]
# (dtype, M, C, [ld, channel offset] of x / dy / add / out): channel slices of wider buffers, offsets multiples of 8
# channels; the last one is the c5 half of the c4|c5 concat buffer (ld = 3072)
LAYOUTS = [(dt, M, C, lay) for dt in ("float32", "bfloat16") for (M, C, lay) in [
    (5000, 64, [(96, 32), (128, 8), (64, 0), (72, 8)]),
    (517, 144, [(208, 64), (144, 0), (152, 8), (160, 16)]),
    (200, 1024, [(3072, 2048), (1024, 0), (3072, 1024), (3072, 2048)])]]


def _id(case):
    return "%s-M%d-C%d" % (("fp32" if case[0] == "float32" else "bf16"), case[1], case[2])


def _gen(case, salt=0):
    import torch
    g = torch.Generator(device=DEV)
    g.manual_seed(1000003 * case[1] + 7919 * case[2] + (17 if case[0] == "float32" else 31) + salt)
    return g


def _randn(g, M, C, dt, mean=0.0, std=1.0):
    import torch
    t = torch.randn(M, C, generator=g, device=DEV) * std
    if not isinstance(mean, float) or mean != 0.0:
        t = t + mean
    return t.to(_dt(dt))


def _chan(g, C, lo, hi):
    import torch
    return torch.rand(C, generator=g, device=DEV) * (hi - lo) + lo


def _slice_of(t, ld, off):
    """t copied into columns [off, off + C) of a NaN-filled [M, ld] buffer -> (buffer, view)"""
    import torch
    M, C = t.shape
    buf = torch.full((M, ld), float("nan"), device=t.device, dtype=t.dtype)
    buf[:, off:off + C] = t
    return buf, buf[:, off:off + C]


def _sentinel_intact(buf, off, C):
    import torch
    return bool(torch.isnan(buf[:, :off]).all()) and bool(torch.isnan(buf[:, off + C:]).all())


def _chunks(M):
    for r in range(0, M, CHUNK):
        yield slice(r, min(M, r + CHUNK))


def _K(M):
    return (4.0 + math.sqrt(M)) * 2.0 ** -24


def _act64(y, relu):
    if relu:
        y = y.clamp(min=0)
    if relu == 2:
        y = y.clamp(max=6)
    return y


def _stats64(x):
    """float64 (mean, biased var, E|x|, E[x^2]) of the stored x, two passes, in chunks"""
    import torch
    M, C = x.shape
    s = torch.zeros(C, dtype=torch.float64, device=x.device)
    sa, sq = s.clone(), s.clone()
    for sl in _chunks(M):
        X = x[sl].double()
        s += X.sum(0); sa += X.abs().sum(0); sq += (X * X).sum(0)
    mean = s / M
    v = torch.zeros_like(s)
    for sl in _chunks(M):
        d = x[sl].double() - mean
        v += (d * d).sum(0)
    return mean, v / M, sa / M, sq / M


def _sums64(x):
    import torch
    M, C = x.shape
    s = torch.zeros(2 * C, dtype=torch.float64, device=x.device)
    for sl in _chunks(M):
        X = x[sl].double()
        s[:C] += X.sum(0); s[C:] += (X * X).sum(0)
    return s


# ------------------------------------------------------------------------------------------------ pointwise kernels
@pytest.mark.parametrize("case", GRID, ids=_id)
def test_affine_act(case):
    import torch
    from sniper_b200 import ops
    dt, M, C = case
    g = _gen(case)
    x = _randn(g, M, C, dt, 0.5, 2.0)
    scale = _chan(g, C, 0.5, 1.5) * torch.where(_chan(g, C, 0, 1) > 0.3, 1.0, -1.0)
    shift = _chan(g, C, -3, 6)
    if M > 1:
        x[1] = ((6.0 - shift) / scale).to(x.dtype)          # pre-activations on / next to the upper clip value
    for relu in (0, 1, 2):
        y = ops.affine_act(x, scale, shift, relu=relu)
        ref = _act64(x.double() * scale.double() + shift.double(), relu)
        _within("affine_act " + dt, y, ref, _ulp_bound(ref, y.dtype))
    y = ops.affine_act(x.clone(), scale, shift, relu=1)
    xin = x.clone()
    assert ops.affine_act(xin, scale, shift, relu=1, out=xin) is xin and torch.equal(xin, y)      # in place


@pytest.mark.parametrize("case", GRID, ids=_id)
def test_cast_add_relu_bwd(case):
    import torch
    from sniper_b200 import ops
    dt, M, C = case
    g = _gen(case, 1)
    a, b = _randn(g, M, C, dt, 0.0, 3.0), _randn(g, M, C, dt, 0.1, 1.0)
    a[0, :4] = 0.0                                                   # relu_bwd: y == 0 passes no gradient
    for to in ("float32", "bfloat16"):
        assert torch.equal(ops.cast_rows(a, dtype=_dt(to)), a.to(_dt(to))), "cast %s -> %s" % (dt, to)
    s = ops.add_rows(a, b)
    ref = a.double() + b.double()
    if dt == "float32":
        assert torch.equal(s, a + b)
    _within("add_rows " + dt, s, ref, _ulp_bound(ref, s.dtype))
    acc = a.clone()
    assert ops.add_rows(acc, b, out=acc) is acc and torch.equal(acc, s)                          # out aliases a
    dx = ops.relu_bwd(a, b)
    assert torch.equal(dx, torch.where(a > 0, b, torch.zeros_like(b)))
    bb = b.clone()
    assert torch.equal(ops.relu_bwd(a, bb, out=bb), dx)                                          # in place over dy


@pytest.mark.parametrize("case", [c for c in SMALL if c[0] == "float32"], ids=_id)
def test_affine_relu_bwd(case):
    """dx = dy * scale * (x * scale + shift > 0) (+ add): two fp32 roundings (the product, the sum)."""
    import torch
    from sniper_b200 import ops
    dt, M, C = case
    g = _gen(case, 2)
    x, dy, add = _randn(g, M, C, dt, 0.5, 2.0), _randn(g, M, C, dt), _randn(g, M, C, dt)
    scale, shift = _chan(g, C, 0.5, 1.5), _chan(g, C, -1, 1)
    X, S, T = x.double(), scale.double(), shift.double()
    y = X * S + T
    amb = y.abs() <= E32 * (X.abs() * S + T.abs())
    assert int(amb.sum()) <= 1e-4 * amb.numel() + 1
    for relu in (0, 1):
        for ad in (None, add):
            dx = ops.affine_relu_bwd(x, dy, scale, shift, add=ad, relu=bool(relu))
            p = dy.double() * S * ((y > 0) if relu else torch.ones_like(y, dtype=torch.bool))
            ref = p if ad is None else p + ad.double()
            bound = E32 * (p.abs() + ref.abs()) + 2.0 ** -149
            _within("affine_relu_bwd", dx, ref, bound, skip=amb if relu else None)


@pytest.mark.parametrize("dt", ["float32", "bfloat16"])
@pytest.mark.parametrize("NB,H,W,C", [(2, 18, 22, 64), (3, 17, 23, 24), (1, 1, 9, 8), (2, 9, 1, 16), (1, 1, 1, 8),
                                      (2, 2, 2, 144), (1, 255, 3, 12)])
def test_maxpool(dt, NB, H, W, C):
    import torch
    import torch.nn.functional as F
    from sniper_b200 import ops
    g = _gen((dt, H * W, C), 3)
    x = _randn(g, NB * H * W, C, dt).view(NB, H, W, C)
    y = ops.maxpool3x3s2(x)
    ref = F.max_pool2d(x.float().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).to(x.dtype)
    assert y.shape == ref.shape and torch.equal(y, ref)


@pytest.mark.parametrize("case", LAYOUTS, ids=_id)
def test_strided_views_are_accepted_and_stay_inside(case):
    """Channel slices of wider buffers for every operand independently: accepted by the argument checks, correct, and
    the columns of the output buffer outside the slice still hold their NaN sentinel."""
    import torch
    from sniper_b200 import ops
    dt, M, C, lay = case
    g = _gen(case, 4)
    x, dy, add = _randn(g, M, C, dt, 0.5, 2.0), _randn(g, M, C, dt), _randn(g, M, C, dt)
    scale, shift = _chan(g, C, 0.5, 1.5), _chan(g, C, -1, 1)
    (_, xv), (_, dyv), (_, addv) = [_slice_of(t, *lay[i]) for i, t in enumerate((x, dy, add))]
    ob, ov = _slice_of(torch.zeros_like(x), *lay[3])

    def fresh():
        ov.fill_(float("nan"))
        return ov

    assert torch.equal(ops.affine_act(xv, scale, shift, relu=2, out=fresh()), ops.affine_act(x, scale, shift, relu=2))
    assert _sentinel_intact(ob, lay[3][1], C)
    assert torch.equal(ops.add_rows(xv, dyv, out=fresh()), ops.add_rows(x, dy)) and _sentinel_intact(ob, lay[3][1], C)
    assert torch.equal(ops.relu_bwd(xv, dyv, out=fresh()), ops.relu_bwd(x, dy)) and _sentinel_intact(ob, lay[3][1], C)
    other = torch.bfloat16 if dt == "float32" else torch.float32
    cb, cv = _slice_of(torch.zeros(M, C, device=DEV, dtype=other), *lay[3])
    assert torch.equal(ops.cast_rows(xv, out=cv), x.to(other)) and _sentinel_intact(cb, lay[3][1], C)
    a, b = ops.BNState(C, DEV), ops.BNState(C, DEV)
    for st in (a, b):
        st.gamma.copy_(scale); st.beta.copy_(shift)
        st.dgamma, st.dbeta = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    ops.bn_stats(x, a); ops.bn_stats(xv, b)
    for f in ("mean", "invstd", "scale", "shift", "moving_mean", "moving_var"):
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    b.sums_f.copy_(_sums64(x)); a.sums_f.copy_(b.sums_f)
    assert torch.equal(ops.bn_apply_train(xv, b, relu=2, out=fresh()), ops.bn_apply_train(x, a, relu=2))
    assert _sentinel_intact(ob, lay[3][1], C)
    for act in (1, 2, 3):
        ref = ops.bn_act_bwd(x, dy, a, act, add=add)
        assert torch.equal(ops.bn_act_bwd(xv, dyv, b, act, add=addv, out=fresh()), ref)
        assert _sentinel_intact(ob, lay[3][1], C)
    assert torch.equal(a.dgamma, b.dgamma) and torch.equal(a.dbeta, b.dbeta)
    # in place, as the residual backward does it: dx over dy, and dx over add
    d2, a2 = dy.clone(), add.clone()
    ref = ops.bn_act_bwd(x, dy, a, 1, add=add)
    assert torch.equal(ops.bn_act_bwd(x, d2, a, 1, add=add, out=d2), ref)
    assert torch.equal(ops.bn_act_bwd(x, dy, a, 1, add=a2, out=a2), ref)
    if dt == "float32":
        assert torch.equal(ops.affine_relu_bwd(xv, dyv, scale, shift, add=addv, out=fresh()),
                           ops.affine_relu_bwd(x, dy, scale, shift, add=add)) and _sentinel_intact(ob, lay[3][1], C)


# ------------------------------------------------------------------------------------------------ statistics
def _regime(g, M, C, dt, regime):
    import torch
    if regime == "std2":
        return _randn(g, M, C, dt, 0.5, 2.0)
    if regime == "mean100std":        # |mean| = 100 std: E[x^2] - E[x]^2 cancels four digits
        sign = torch.where(_chan(g, C, 0, 1) > 0.5, 1.0, -1.0)
        return _randn(g, M, C, dt, 70.0 * sign, 0.7)
    k = (torch.arange(C, device=DEV) % 27 - 13).float() / 4       # constant columns, exactly summable in fp32
    return k.expand(M, C).to(_dt(dt)).contiguous()


def _check_stats(tag, x, bn, M, gamma, beta, mm0, mv0, momentum, fix_gamma, update_moving, regime, exact_sums):
    """bn.(mean, invstd, scale, shift, moving_*) against the float64 statistics of the stored x.  exact_sums: the sums
    were float64 to begin with (finalize / fused apply), so only the final fp32 roundings remain."""
    import torch
    mean, var, ea, e2 = _stats64(x)
    k = 2.0 ** -50 if exact_sums else _K(M)
    t_mean = k * ea + 2.0 ** -24 * mean.abs() + 2.0 ** -149
    _within(tag + " mean", bn.mean, mean, t_mean)
    if regime == "const":
        assert torch.equal(bn.mean.double(), mean) and bool((var == 0).all())
        is_exact = torch.full_like(bn.invstd, 1.0 / math.sqrt(float(torch.tensor(EPS, dtype=torch.float32))))
        assert torch.equal(bn.invstd, is_exact), "var = 0 must publish invstd = 1 / sqrt(eps)"
    # var = E[x^2] - m^2: both terms carry k * E[x^2] (|m| E|x| <= E[x^2]), plus double rounding of the difference
    t_var = 3 * k * e2 + 2.0 ** -50 * e2
    eps32 = float(torch.tensor(EPS, dtype=torch.float32))
    inv = 1.0 / torch.sqrt(var + eps32)
    t_is = inv * (0.5 * t_var / (var + eps32) + 2.0 ** -23)
    _within(tag + " invstd", bn.invstd, inv, t_is)
    var_k = 1.0 / bn.invstd.double() ** 2 - eps32
    ok = var > 0
    if bool(ok.any()) and M > 1:
        rel = ((var_k - var).abs() / var)[ok]
        lim = (t_var / var + 2.0 ** -21 * (var + eps32) / var)[ok]
        _note(tag + " var, relative (%s)" % regime, rel, lim)
        assert bool((rel <= lim).all())
        if M >= 1000:
            assert float(rel.max()) <= 1e-3, "relative variance error %.3e in regime %s" % (float(rel.max()), regime)
    gm = torch.ones_like(gamma) if fix_gamma else gamma
    assert torch.equal(bn.scale, gm * bn.invstd), "scale must be gamma * invstd in fp32 (invstd itself with fix_gamma)"
    sh = beta.double() - bn.mean.double() * gm.double() * bn.invstd.double()
    _within(tag + " shift", bn.shift, sh, 3 * 2.0 ** -24 * (beta.double().abs() + (beta.double() - sh).abs()) + 2.0 ** -149)
    if update_moving:
        unb = var * M / (M - 1) if M > 1 else var
        momentum = float(torch.tensor(momentum, dtype=torch.float32))      # the kernel's fp32 momentum; 1 - it is exact
        rm = mm0.double() * momentum + mean * (1 - momentum)
        rv = mv0.double() * momentum + unb * (1 - momentum)
        _within(tag + " moving_mean", bn.moving_mean, rm, t_mean + E32 * (mm0.double().abs() + mean.abs()))
        _within(tag + " moving_var", bn.moving_var, rv, 1.1 * t_var + E32 * (mv0.double().abs() + unb.abs()))
    else:
        assert torch.equal(bn.moving_mean, mm0) and torch.equal(bn.moving_var, mv0), "moving statistics were touched"


def _bn_state(g, C, pool=None):
    from sniper_b200 import ops
    import torch
    bn = ops.BNState(C, DEV, pool=pool)
    if pool is not None:
        return bn
    _fill_bn(g, bn)
    return bn


def _fill_bn(g, bn):
    C = bn.C
    bn.gamma.copy_(_chan(g, C, 0.5, 1.5)); bn.beta.copy_(_chan(g, C, -1, 1))
    bn.moving_mean.copy_(_chan(g, C, -1, 1)); bn.moving_var.copy_(_chan(g, C, 0.5, 2))


@pytest.mark.parametrize("regime", ["std2", "mean100std", "const"])
@pytest.mark.parametrize("case", SMALL, ids=_id)
def test_bn_stats(case, regime):
    import torch
    from sniper_b200 import ops
    dt, M, C = case
    g = _gen(case, 5)
    x = _regime(g, M, C, dt, regime)
    for fix_gamma, update_moving in ((False, True), (True, False)):
        bn = _bn_state(g, C)
        mm0, mv0 = bn.moving_mean.clone(), bn.moving_var.clone()
        ops.bn_stats(x, bn, eps=EPS, momentum=0.9, fix_gamma=fix_gamma, update_moving=update_moving)
        assert float(bn.sums.abs().sum()) == 0.0                                   # scratch left zeroed
        _check_stats("bn_stats " + dt, x, bn, M, bn.gamma, bn.beta, mm0, mv0, 0.9, fix_gamma, update_moving, regime, False)
        again = _bn_state(_gen(case, 5), C)
        again.gamma.copy_(bn.gamma); again.beta.copy_(bn.beta)
        ops.bn_stats(x, again, eps=EPS, momentum=0.9, fix_gamma=fix_gamma, update_moving=False)
        for f in ("mean", "invstd", "scale", "shift"):                              # run to run: bit-identical
            assert torch.equal(getattr(bn, f), getattr(again, f)), f


@pytest.mark.parametrize("case", GRID, ids=_id)
def test_bn_apply_train_is_finalize_then_affine_act(case):
    """Fused finalise + apply == bn_finalize + affine_act bit for bit over the whole grid, for every activation code and
    both flags; with the state taken from a BNPool (vectors packed back to back) nothing outside the state's own six
    vectors changes -- a ragged last slab must not publish channels >= C into the next layer's vectors."""
    import torch
    from sniper_b200 import ops
    dt, M, C = case
    g = _gen(case, 6)
    x = _randn(g, M, C, dt, 0.3, 1.5)
    sums = _sums64(x)
    pool = ops.BNPool(C + 16, DEV)
    before, b, after = ops.BNState(8, DEV, pool=pool), ops.BNState(C, DEV, pool=pool), ops.BNState(8, DEV, pool=pool)
    pool.finalize()
    pool.f.copy_(torch.rand(pool.f.shape, generator=g, device=DEV) + 0.5)
    base = pool.f.data_ptr()
    own = torch.zeros(pool.f.numel(), dtype=torch.bool, device=DEV)
    for f in ("mean", "invstd", "scale", "shift", "moving_mean", "moving_var"):
        o = (getattr(b, f).data_ptr() - base) // 4
        own[o:o + C] = True
    for relu, fix_gamma, update_moving in ((1, False, True), (2, True, True), (0, False, False)):
        a = _bn_state(g, C)
        a.gamma.copy_(b.gamma); a.beta.copy_(b.beta); a.moving_mean.copy_(b.moving_mean); a.moving_var.copy_(b.moving_var)
        mm0, mv0 = a.moving_mean.clone(), a.moving_var.clone()
        a.sums.copy_(sums); b.sums_f.copy_(sums)
        snap = pool.f.clone()
        ops.bn_finalize(a, M, eps=EPS, momentum=0.9, fix_gamma=fix_gamma, update_moving=update_moving)
        ya = ops.affine_act(x, a.scale, a.shift, relu=relu)
        yb = ops.bn_apply_train(x, b, eps=EPS, momentum=0.9, relu=relu, fix_gamma=fix_gamma, update_moving=update_moving)
        assert torch.equal(ya, yb)
        for f in ("mean", "invstd", "scale", "shift", "moving_mean", "moving_var"):
            assert torch.equal(getattr(a, f), getattr(b, f)), f
        assert torch.equal(b.sums_f, sums) and float(a.sums.abs().sum()) == 0.0
        assert torch.equal(pool.f[~own], snap[~own]), "a vector of a neighbouring layer was written"
        assert float(before.sums_f.abs().sum()) == 0.0 and float(after.sums_f.abs().sum()) == 0.0
        if fix_gamma:
            assert torch.equal(b.scale, b.invstd)
        _check_stats("bn_finalize " + dt, x, a, M, a.gamma, a.beta, mm0, mv0, 0.9, fix_gamma, update_moving, "std2", True)
        ref = _act64(x.double() * a.scale.double() + a.shift.double(), relu)
        _within("bn_apply_train y " + dt, yb, ref, _ulp_bound(ref, yb.dtype))
    assert before.C == after.C == 8


# ------------------------------------------------------------------------------------------------ backward
def _check_bwd(tag, x, dy, add, bn, act, dx, dgamma0, dbeta0, defer):
    """dx, dgamma, dbeta (or the deferred sums) of act(bn_train(x)) against float64 statistics of the stored x."""
    import torch
    M, C = x.shape
    mean, var, _, _ = _stats64(x)
    eps32 = float(torch.tensor(EPS, dtype=torch.float32))
    inv = 1.0 / torch.sqrt(var + eps32)
    gm, bt = bn.gamma.double(), bn.beta.double()
    sc, sh = gm * inv, bt - mean * gm * inv
    # what the kernel's own statistics add to the comparison (measured, not assumed)
    dsc, dsh = (bn.scale.double() - sc).abs(), (bn.shift.double() - sh).abs()
    dmean, dinv = (bn.mean.double() - mean).abs(), (bn.invstd.double() - inv).abs()
    z = lambda: torch.zeros(C, dtype=torch.float64, device=x.device)
    S1, S2, A1, A2, T1, T2, namb = z(), z(), z(), z(), z(), z(), 0

    def parts(sl):
        X, G = x[sl].double(), dy[sl].double()
        y = X * sc + sh
        tol = X.abs() * dsc + dsh + E32 * (X.abs() * sc.abs() + sh.abs())
        if act == 1:
            mask, amb = y > 0, y.abs() <= tol
        elif act == 2:
            mask, amb = (y >= 0) & (y <= 6), (y.abs() <= tol) | ((y - 6).abs() <= tol)
        else:
            mask, amb = torch.ones_like(y, dtype=torch.bool), torch.zeros_like(y, dtype=torch.bool)
        xhat = (X - mean) * inv
        dxh = dmean * inv + (X - mean).abs() * dinv + 2.0 ** -22 * (X.abs() + mean.abs()) * inv
        return G * mask, xhat, dxh, amb, G.abs()

    for sl in _chunks(M):
        Gm, xhat, dxh, amb, Ga = parts(sl)
        S1 += Gm.sum(0); S2 += (Gm * xhat).sum(0)
        A1 += (Ga * amb).sum(0); A2 += (Ga * amb * (xhat.abs() + dxh)).sum(0)
        T1 += Gm.abs().sum(0); T2 += (Gm.abs() * xhat.abs()).sum(0) * _K(M) + (Gm.abs() * dxh).sum(0)
        namb += int(amb.sum())
    # (a column of very few rows can have a variance within the fp32 rounding of x^2 of zero; eps then dominates
    # invstd, the published scale legitimately differs from float64 by percents and the test has no power there)
    assert M < 32 or namb <= 1e-4 * x.numel() + 1, "%d of %d mask elements are ambiguous" % (namb, x.numel())
    t1 = _K(M) * T1 + A1 + 2.0 ** -149
    t2 = T2 + A2 + 2.0 ** -149
    for sl in _chunks(M):
        Gm, xhat, dxh, amb, _ = parts(sl)
        inner = Gm - S1 / M - xhat * (S2 / M)
        ref = sc * inner
        mag = sc.abs() * (Gm.abs() + S1.abs() / M + (xhat * S2 / M).abs())
        bound = sc.abs() * (t1 / M + xhat.abs() * t2 / M + dxh * (S2.abs() + t2) / M) + dsc * inner.abs() + 6 * 2.0 ** -24 * mag
        if add is not None:
            ref = ref + add[sl].double()
            bound = bound + 2.0 ** -24 * (mag + ref.abs())
        if dx.dtype == torch.bfloat16:
            bound = bound + ref.abs() * BF * 1.01 + 1e-6
        else:
            bound = bound + 2.0 ** -149
        _within(tag + " dx", dx[sl], ref, bound, skip=amb)
    if defer:
        assert torch.equal(bn.dgamma, dgamma0) and torch.equal(bn.dbeta, dbeta0), "deferred: gradients must be untouched"
        _within(tag + " deferred sum(g)", bn.sums[:C], S1, t1)
        _within(tag + " deferred sum(g xhat)", bn.sums[C:], S2, t2)
    else:
        assert float(bn.sums.abs().sum()) == 0.0
        _within(tag + " dbeta", bn.dbeta, dbeta0.double() + S1, t1 + E32 * (dbeta0.double().abs() + S1.abs()))
        _within(tag + " dgamma", bn.dgamma, dgamma0.double() + S2, t2 + E32 * (dgamma0.double().abs() + S2.abs()))
    return S1, S2, t1, t2


@pytest.mark.parametrize("case", SMALL, ids=_id)
def test_bn_act_bwd(case):
    import torch
    from sniper_b200 import ops
    dt, M, C = case
    g = _gen(case, 7)
    x, dy, add = _randn(g, M, C, dt, 0.5, 2.0), _randn(g, M, C, dt), _randn(g, M, C, dt)
    bn = _bn_state(g, C)
    ops.bn_stats(x, bn, eps=EPS)
    for act in (1, 2, 3):
        for ad in (None, add):
            for defer in (False, True):
                bn.dgamma, bn.dbeta = _chan(g, C, -2, 2), _chan(g, C, -2, 2)       # the gradients ACCUMULATE
                g0, b0 = bn.dgamma.clone(), bn.dbeta.clone()
                dx = ops.bn_act_bwd(x, dy, bn, act, add=ad, defer=defer)
                S1, S2, t1, t2 = _check_bwd("bn_act_bwd " + dt, x, dy, ad, bn, act, dx, g0, b0, defer)
                if act == 1 and ad is None and not defer:
                    assert torch.equal(ops.bn_relu_bwd(x, dy, bn), dx), "two runs differ"        # run to run
                    assert float(bn.sums.abs().sum()) == 0.0
                if defer:
                    bn.sums.zero_()
    # one batched parameter-gradient launch over deferred states of different widths
    states, want = [], []
    for i, Ci in enumerate((C, 8, 2048, 24)):
        gi = _gen((dt, 37, Ci), 8 + i)
        st = _bn_state(gi, Ci)
        xi, di = _randn(gi, 37, Ci, dt, 0.5, 2.0), _randn(gi, 37, Ci, dt)
        ops.bn_stats(xi, st, eps=EPS)
        st.dgamma, st.dbeta = _chan(gi, Ci, -2, 2), _chan(gi, Ci, -2, 2)
        g0, b0 = st.dgamma.clone(), st.dbeta.clone()
        ops.bn_act_bwd(xi, di, st, 1, defer=True)
        st.sums_f.fill_(3.0)
        states.append(st); want.append((g0 + st.sums[Ci:].float(), b0 + st.sums[:Ci].float()))
    ops.bn_param_grad_batched(ops.bn_param_grad_jobs(states, DEV))
    for st, (wg, wb) in zip(states, want):
        assert torch.equal(st.dgamma, wg) and torch.equal(st.dbeta, wb)
        assert float(st.sums.abs().sum()) == 0.0 and float(st.sums_f.abs().sum()) == 0.0


@pytest.mark.parametrize("dt", ["float32", "bfloat16"])
def test_clip_mask_boundaries(dt):
    """Pre-activations exactly on and one storage ulp either side of 0 and 6 (scale 1, shift 0, mean 0, invstd 1, so the
    kernel's fma reproduces x exactly): ReLU passes y > 0, clip passes 0 <= y <= 6 (both ends included), forward and
    backward agree, and a wrong side shows as an O(1) error in dx and in the sums."""
    import torch
    from sniper_b200 import ops
    M, C = 64, 32
    t = _dt(dt)
    g = _gen((dt, M, C), 10)
    edge = torch.tensor([0.0, 6.0], device=DEV, dtype=t)
    vals = torch.cat([edge, torch.nextafter(edge, edge + 1), torch.nextafter(edge, edge - 1), -edge])     # 8 values
    idx = (torch.arange(M, device=DEV)[:, None] + torch.arange(C, device=DEV)[None, :]) % 8
    x = vals[idx]                                             # every column holds all eight values
    dy = _randn(g, M, C, dt) + 3.0
    bn = ops.BNState(C, DEV)
    bn.scale.fill_(1.0); bn.invstd.fill_(1.0)                 # mean = shift = 0: y = xhat = x exactly
    X, G = x.double(), dy.double()
    for act, mask in ((1, X > 0), (2, (X >= 0) & (X <= 6))):
        fwd = ops.affine_act(x, bn.scale, bn.shift, relu=act)
        assert torch.equal(fwd, _act64(X, act).to(t))
        assert torch.equal(mask, (fwd.double() == X) & ((X != 0) | (act == 2)) | ((X == 0) & (act == 2)))
        bn.dgamma, bn.dbeta = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
        dx = ops.bn_act_bwd(x, dy, bn, act)
        Gm = G * mask
        S1, S2 = Gm.sum(0), (Gm * X).sum(0)
        ref = Gm - S1 / M - X * (S2 / M)
        mag = Gm.abs() + S1.abs() / M + (X * S2 / M).abs()
        bound = 1e-5 * mag + (ref.abs() * BF * 1.01 + 1e-6 if dt == "bfloat16" else 2.0 ** -149)
        _within("clip boundaries dx " + dt, dx, ref, bound)
        _within("clip boundaries dbeta " + dt, bn.dbeta, S1, 1e-5 * Gm.abs().sum(0) + 1e-30)
        _within("clip boundaries dgamma " + dt, bn.dgamma, S2, 1e-5 * (Gm * X).abs().sum(0) + 1e-30)


@pytest.mark.parametrize("dt", ["float32", "bfloat16"])
def test_stem_shape(dt):
    """The real first-layer shape of a 20-chip step: 1 310 720 rows x 64 channels, where each thread of the statistics
    kernel adds ~150 values in fp32 before the double reduction; the second regime has |mean| = 100 std."""
    import torch
    from sniper_b200 import ops
    M, C = STEM
    case = (dt, M, C)
    g = _gen(case, 9)
    for regime in ("std2", "mean100std"):
        x = _regime(g, M, C, dt, regime)
        bn = _bn_state(g, C)
        mm0, mv0 = bn.moving_mean.clone(), bn.moving_var.clone()
        ops.bn_stats(x, bn, eps=EPS, momentum=0.9)
        _check_stats("stem bn_stats " + dt, x, bn, M, bn.gamma, bn.beta, mm0, mv0, 0.9, False, True, regime, False)
    b2 = _bn_state(g, C)
    b2.gamma.copy_(bn.gamma); b2.beta.copy_(bn.beta)
    b2.sums_f.copy_(_sums64(x))
    y = ops.bn_apply_train(x, b2, eps=EPS, relu=True)
    for sl in _chunks(M):
        ref = _act64(x[sl].double() * b2.scale.double() + b2.shift.double(), 1)
        _within("stem bn_apply_train y " + dt, y[sl], ref, _ulp_bound(ref, y.dtype))
    del y
    x = _regime(g, M, C, dt, "std2")
    ops.bn_stats(x, bn, eps=EPS)
    dy = _randn(g, M, C, dt)
    bn.dgamma, bn.dbeta = _chan(g, C, -2, 2), _chan(g, C, -2, 2)
    g0, b0 = bn.dgamma.clone(), bn.dbeta.clone()
    dx = ops.bn_act_bwd(x, dy, bn, 1)
    _check_bwd("stem bn_act_bwd " + dt, x, dy, None, bn, 1, dx, g0, b0, False)


def test_zz_report():
    """Worst error per assertion class over this run, as a fraction of its bound (pytest -s shows it)."""
    print()
    for what in sorted(WORST):
        r, e, b = WORST[what]
        print("  %-44s worst error / bound %.3f   (error %.3e, bound %.3e)" % (what, r, e, b))
    assert all(r[0] <= 1.0 for r in WORST.values())
