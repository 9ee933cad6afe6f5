"""Loss layers (csrc/losses.cu) and the FocusPixel accuracy counter against float64.

Bounds.  A probability is exp(x - m) / sum: the fp32 difference x - m carries 2^-24 |x - m| (an error of |x - m| / 2 ulp
in the exponential), expf 2 ulp, the sum of K terms (K / 32 per lane + 5 shuffles) and the reciprocal / product the
rest: |p - p64| <= 2^-23 p (4 + K / 64 + |x - m| / 2) + 2^-126 (flush of the exponential).  A gradient is (p - onehot) *
norm and inherits the bound of p (not of the difference, which cancels for a confident correct row) plus 2 ulp of
p + onehot for the fp32 quotient grad_scale / valid, the difference and the product.  loss_sum is a
chain of fp32 additions onto one running total (per thread, then one float atomic per warp; the flat softmax adds one
atomic per valid row), each rounding to 2^-24 of the total: |error| <= adds * 2^-24 * sum|terms| + the per-term error of
log p, with `adds` the longest chain.  A sqrt(adds) bound does NOT hold: rows at the clamp add the same value
-log(1e-14) over and over, and equal addends round the same way (measured on an H100: 6000 x 81 rows, logits scaled by
30, loss_sum 46870.74 against 46871.42 in float64, 1.5e-5 relative, five times the square-root bound).  The loss of a
row whose probability underflows is -log(1e-14), the clamp of the kernels.

Layout conventions exercised with H != W and ld > channels: RPN labels in (a, h, w) order, targets / weights NCHW,
scores / gradients NHWC; totals above 132 * 8 * 256 elements make the grid-stride loops take a second trip."""
import math

import pytest

pytestmark = pytest.mark.gpu

E32 = 2.0 ** -23
CLAMP = 1e-14


def _gen(*key):
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(sum((i + 1) * 7919 * int(k) for i, k in enumerate(key)) + 5)
    return g


def _clamp32():
    import torch
    return float(torch.tensor(CLAMP, dtype=torch.float32))


def _labels(g, shape, hi, mode):
    import torch
    lab = torch.randint(0, hi, shape, generator=g, device="cuda").float()
    if mode == "all_ignored":
        lab.fill_(-1.0)
    elif mode == "mixed":
        lab[torch.rand(shape, generator=g, device="cuda") < 0.3] = -1.0
    return lab


def _softmax64(z):
    """z [..., K] float64 -> (p, |z - max|)"""
    import torch
    m = z.max(-1, keepdim=True).values
    return torch.softmax(z, -1), (z - m).abs()


def _p_bound(p, d, K):
    return E32 * p * (4 + K / 64.0 + d / 2) + 2.0 ** -126


def _chain(total):
    """longest chain of additions of the grid-stride loss kernels: a thread's share + 5 shuffles + one atomic per warp"""
    blocks = min(132 * 8, max(1, (total + 255) // 256))
    return (total + blocks * 256 - 1) // (blocks * 256) + 5 + blocks * 8


def _loss_check(got, terms, extra, adds):
    total = float(terms.sum())
    bound = (2 + adds) * 2.0 ** -24 * float(terms.abs().sum()) + float(extra)
    assert abs(float(got) - total) <= bound, "loss_sum %.9g vs %.9g, bound %.3e" % (float(got), total, bound)


# ------------------------------------------------------------------------------------------------ count_valid
@pytest.mark.parametrize("n", [1, 31, 33, 1000, 20 * 32 * 32 * 21])
@pytest.mark.parametrize("mode", ["mixed", "all_ignored", "none_ignored"])
def test_count_valid(n, mode):
    import torch
    from sniper_b200 import ops
    lab = _labels(_gen(n, len(mode)), (n,), 81, mode)
    cnt = torch.full((1,), 5, dtype=torch.int32, device="cuda")              # accumulates onto what is there
    ops.count_valid(lab, cnt)
    assert int(cnt) == 5 + int((lab != -1).sum())
    c0 = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.count_valid(lab, c0, ignore=0)
    assert int(c0) == int((lab.int() != 0).sum())


# ------------------------------------------------------------------------------------------------ RPN softmax
@pytest.mark.parametrize("scale", [1.0, 30.0, 90.0])
@pytest.mark.parametrize("mode", ["mixed", "all_ignored", "none_ignored"])
@pytest.mark.parametrize("B,H,W,A,wide", [(1, 1, 1, 1, False), (3, 8, 8, 21, True), (20, 32, 32, 21, False),
                                          (2, 7, 5, 15, True), (2, 7, 5, 15, False), (20, 16, 16, 1, True)])
def test_rpn_softmax_loss(B, H, W, A, wide, mode, scale):
    import torch
    from sniper_b200 import ops
    if scale != 1.0 and mode != "mixed":
        pytest.skip("the scales run with mixed labels")
    g = _gen(B, H, W, A, wide, len(mode), scale)
    ld = 128 if wide else 2 * A
    score = torch.randn(B, H, W, ld, generator=g, device="cuda") * scale
    if scale > 1:
        score[..., 0] = 90.0                                   # one column pinned high, its partner low
        score[..., A] = -90.0
    label = _labels(g, (B, A * H * W), 2, mode)
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.count_valid(label, cnt)
    prob = torch.full((B, H, W, 2 * A), float("nan"), device="cuda")
    ds = torch.full((B, H, W, ld), float("nan"), device="cuda")
    loss = torch.zeros(1, device="cuda")
    gs = 0.75
    ops.rpn_softmax_loss(score[..., :2 * A], label, A, gs, cnt, prob, ds[..., :2 * A], loss)
    z = torch.stack([score[..., :A], score[..., A:2 * A]], -1).double()          # [B,H,W,A,2]
    p, d = _softmax64(z)
    pb = _p_bound(p, d, 2)
    got_p = torch.stack([prob[..., :A], prob[..., A:]], -1).double()
    assert bool(torch.isfinite(prob).all()) and bool(((got_p - p).abs() <= pb).all())
    assert bool(((got_p.sum(-1) - 1).abs() <= 4 * E32).all())
    lab = label.view(B, A, H, W).permute(0, 2, 3, 1)                              # (a,h,w) -> [B,H,W,A]
    valid = lab != -1
    norm = gs / max(1, int(valid.sum()))
    onehot = torch.stack([lab == 0, lab == 1], -1).double()
    gref = (p - onehot) * norm * valid.unsqueeze(-1)
    got_g = torch.stack([ds[..., :A], ds[..., A:2 * A]], -1).double()
    assert bool(torch.isfinite(got_g).all())
    assert bool(((got_g - gref).abs() <= (pb + 2 * E32 * (p + onehot)) * norm).all())
    assert bool(torch.isnan(ds[..., 2 * A:]).all()), "columns beyond 2A were written"
    if mode == "all_ignored":
        assert float(got_g.abs().sum()) == 0.0 and float(loss) == 0.0
    pl = (p * onehot).sum(-1)
    terms = -torch.log(pl.clamp(min=_clamp32())) * valid
    dl = ((d * onehot).sum(-1) / 2 + 6) * E32 * valid
    _loss_check(loss, terms, dl.sum(), _chain(B * H * W * A))
    # null gradient (inference: probabilities only), null valid count (norm 1)
    p2 = torch.empty_like(prob)
    ops.rpn_softmax_loss(score[..., :2 * A], label, A, gs, None, p2, None, None)
    assert torch.equal(p2, prob)
    d2 = torch.empty(B, H, W, 2 * A, device="cuda")
    ops.rpn_softmax_loss(score[..., :2 * A], label, A, 1.0, None, p2, d2, None)
    g1 = torch.stack([d2[..., :A], d2[..., A:]], -1).double()
    assert bool(((g1 - (p - onehot) * valid.unsqueeze(-1)).abs() <= pb + 2 * E32 * (p + onehot)).all())


# ------------------------------------------------------------------------------------------------ flat softmax + CE
@pytest.mark.parametrize("scale", [1.0, 30.0, 90.0])
@pytest.mark.parametrize("mode", ["mixed", "all_ignored", "none_ignored"])
@pytest.mark.parametrize("N,K,ld", [(1, 2, 2), (33, 3, 8), (700, 81, 88), (6000, 81, 81), (5, 1000, 1024), (4099, 2, 2)])
def test_softmax_ce(N, K, ld, mode, scale):
    import torch
    from sniper_b200 import ops
    if scale != 1.0 and mode != "mixed":
        pytest.skip("the scales run with mixed labels")
    g = _gen(N, K, ld, len(mode), scale)
    logits = torch.randn(N, ld, generator=g, device="cuda") * scale
    if scale > 1:
        logits[:, 0] = 90.0
        logits[:, K - 1] = -90.0
    label = _labels(g, (N,), K, mode)
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.count_valid(label, cnt)
    prob = torch.full((N, K), float("nan"), device="cuda")
    grad = torch.full((N, ld), float("nan"), device="cuda")
    loss = torch.zeros(1, device="cuda")
    gs = 1.5
    ops.softmax_ce(logits, label, K, gs, cnt, prob, grad, loss)
    p, d = _softmax64(logits[:, :K].double())
    pb = _p_bound(p, d, K)
    assert bool(torch.isfinite(prob).all()) and bool(((prob.double() - p).abs() <= pb).all())
    assert bool(((prob.double().sum(-1) - 1).abs() <= (4 + K / 32.0) * E32).all())
    valid = (label != -1)
    onehot = torch.zeros(N, K, dtype=torch.float64, device="cuda")
    onehot[valid, label[valid].long()] = 1.0
    norm = gs / max(1, int(valid.sum()))
    gref = (p - onehot) * norm * valid.unsqueeze(-1)
    assert bool(torch.isfinite(grad[:, :K]).all())
    assert bool(((grad[:, :K].double() - gref).abs() <= (pb + 2 * E32 * (p + onehot)) * norm).all())
    assert bool(torch.isnan(grad[:, K:]).all()), "columns beyond K were written"
    if mode == "all_ignored":
        assert float(grad[:, :K].abs().sum()) == 0.0 and float(loss) == 0.0
    pl = (p * onehot).sum(-1)
    terms = -torch.log(pl.clamp(min=_clamp32())) * valid
    dl = ((d * onehot).sum(-1) / 2 + 6 + K / 64.0) * E32 * valid
    _loss_check(loss, terms, dl.sum(), int(valid.sum()))
    if scale == 90.0:                          # label rows on the low column: probability underflows, loss = the clamp
        low = valid & (label == K - 1)
        assert bool((terms[low] == -math.log(_clamp32())).all())
    # every optional pointer null in turn (inference passes grad = None; MobileNetV2 passes valid_cnt = None)
    for pr, gr, ls, vc in ((None, None, None, None), (torch.empty_like(prob), None, torch.zeros(1, device="cuda"), cnt),
                           (None, torch.empty_like(grad), None, None)):
        ops.softmax_ce(logits, label, K, gs, vc, pr, gr, ls)
        if pr is not None:
            assert torch.equal(pr, prob)
        if gr is not None:
            assert bool(((gr[:, :K].double() - (p - onehot) * gs * valid.unsqueeze(-1)).abs()
                         <= (pb + 2 * E32 * (p + onehot)) * gs).all())
        if ls is not None:
            _loss_check(ls, terms, dl.sum(), int(valid.sum()))


# ------------------------------------------------------------------------------------------------ smooth L1
def _sl1_64(d):
    import torch
    a = d.abs()
    return torch.where(a < 1, 0.5 * d * d, a - 0.5), torch.where(a < 1, d, torch.sign(d))


@pytest.mark.parametrize("N,C,ld", [(1, 4, 4), (33, 4, 88), (700, 4, 88), (6000, 81, 96), (5, 1000, 1000)])
def test_smooth_l1_loss(N, C, ld):
    import torch
    from sniper_b200 import ops
    g = _gen(N, C, ld)
    buf = torch.randn(N, ld, generator=g, device="cuda") * 2
    off = ld - C if ld >= 2 * C else 0
    pred = buf[:, off:off + C]
    target = torch.randn(N, C, generator=g, device="cuda")
    weight = (torch.rand(N, C, generator=g, device="cuda") > 0.4).float() * torch.rand(N, C, generator=g, device="cuda")
    gbuf = torch.full((N, ld), float("nan"), device="cuda")
    loss = torch.zeros(1, device="cuda")
    gs = 1.0 / 3008
    ops.smooth_l1_loss(pred, target, weight, C, gs, gbuf[:, off:off + C], loss)
    d32 = (pred - target)                                       # the fp32 difference the kernel forms decides the branch
    val, der = _sl1_64(d32.double())
    gref = weight.double() * der * gs
    got = gbuf[:, off:off + C].double()
    assert bool(((got - gref).abs() <= 2 * E32 * gref.abs() + 2.0 ** -149).all())
    assert bool(torch.isnan(gbuf[:, :off]).all()) and bool(torch.isnan(gbuf[:, off + C:]).all())
    _loss_check(loss, weight.double() * val, 3 * E32 * float((weight.double() * val).sum()), _chain(N * C))
    z = torch.zeros(1, device="cuda")
    g0 = torch.empty(N, C, device="cuda")
    ops.smooth_l1_loss(pred, target, torch.zeros_like(weight), C, gs, g0, z)           # zero weights
    assert float(g0.abs().sum()) == 0.0 and float(z) == 0.0
    ops.smooth_l1_loss(pred, target, weight, C, gs, g0, None)                           # null loss_sum
    assert torch.equal(g0, gbuf[:, off:off + C])


def test_smooth_l1_kink_sides():
    """|d| < 1 is the quadratic branch: d = 1 exactly and one step above give gradient +-1 (times weight * scale), one
    step below gives d itself."""
    import torch
    from sniper_b200 import ops
    one = torch.tensor(1.0, device="cuda")
    below, above = torch.nextafter(one, one * 0), torch.nextafter(one, one * 2)
    d = torch.stack([one, below, above, -one, -below, -above, one * 0, one * 0]).view(2, 4)
    grad, loss = torch.empty(2, 4, device="cuda"), torch.zeros(1, device="cuda")
    ops.smooth_l1_loss(d, torch.zeros_like(d), torch.ones_like(d), 4, 1.0, grad, loss)
    want = torch.stack([one, below, one, -one, -below, -one, one * 0, one * 0]).view(2, 4)
    assert torch.equal(grad, want)
    ref = float((0.5 + 0.5 * below.double() ** 2 + (above.double() - 0.5)) * 2)
    assert abs(float(loss) - ref) <= 8 * 2.0 ** -24 * ref


@pytest.mark.parametrize("B,H,W,A,wide", [(1, 1, 1, 1, False), (3, 8, 8, 21, True), (20, 32, 32, 21, False),
                                          (2, 7, 5, 15, True)])
def test_rpn_smooth_l1_loss(B, H, W, A, wide):
    import torch
    from sniper_b200 import ops
    g = _gen(B, H, W, A, wide, 3)
    C4 = 4 * A
    ld = 128 if wide else C4
    pred = torch.randn(B, H, W, ld, generator=g, device="cuda") * 2
    target = torch.randn(B, C4, H, W, generator=g, device="cuda")               # NCHW, the iterator's layout
    weight = (torch.rand(B, C4, H, W, generator=g, device="cuda") > 0.7).float()
    dp = torch.full((B, H, W, ld), float("nan"), device="cuda")
    loss = torch.zeros(1, device="cuda")
    ops.rpn_smooth_l1_loss(pred, target, weight, C4, 0.25, dp, loss)
    t, w = target.permute(0, 2, 3, 1), weight.permute(0, 2, 3, 1)
    d32 = pred[..., :C4] - t
    val, der = _sl1_64(d32.double())
    gref = w.double() * der * 0.25
    assert bool(((dp[..., :C4].double() - gref).abs() <= 2 * E32 * gref.abs() + 2.0 ** -149).all())
    assert bool(torch.isnan(dp[..., C4:]).all())
    _loss_check(loss, w.double() * val, 3 * E32 * float((w.double() * val).sum()), _chain(B * H * W * C4))
    d2 = torch.empty(B, H, W, C4, device="cuda")
    ops.rpn_smooth_l1_loss(pred, target, weight, C4, 0.25, d2, None)
    assert torch.equal(d2, dp[..., :C4])


# ------------------------------------------------------------------------------------------------ FocusPixel accuracy
@pytest.mark.parametrize("n,ldp", [(1, 2), (33, 2), (20 * 32 * 32, 2), (20 * 32 * 32, 8), (132 * 4 * 256 + 77, 2)])
def test_focus_acc(n, ldp):
    """hits = #(argmax == label) with ties going to channel 0, valid = #(label != -1); exact integers, accumulated."""
    import torch
    from sniper_b200 import ops
    g = _gen(n, ldp)
    prob = torch.rand(n, ldp, generator=g, device="cuda")
    prob[::5, 1] = prob[::5, 0]                                                   # ties
    label = _labels(g, (n,), 2, "mixed")
    counts = torch.tensor([3.0, 7.0], device="cuda")
    ops.focus_acc(prob, label, counts)
    valid = label != -1
    pred = (prob[:, 1] > prob[:, 0]).float()
    assert counts.tolist() == [3.0 + int(((pred == label) & valid).sum()), 7.0 + int(valid.sum())]
    c2 = torch.zeros(2, device="cuda")
    ops.focus_acc(prob, torch.full((n,), -1.0, device="cuda"), c2)
    assert c2.tolist() == [0.0, 0.0]
