"""The fused SGD-momentum update (sniper_sgd_mom, sniper_sgd_mom_dev) against float64.

Reference: mom' = momentum * mom - lr * wd * w - lr * rescale * g;  w' = w + mom', evaluated in float64 from the fp32
inputs with the fp32 products lr = hyper[0] * lr_mult, wd = hyper[1] * wd_mult, lr * wd and lr * rescale the kernel forms
first.  mom' carries at most half an ulp on momentum * mom, one ulp on each of the two products with a pre-rounded
factor and two half ulps on the two sums: |error| <= 2 * 2^-23 * sum|terms|.  w' is ONE fp32 addition of the kernel's own
mom', so it must equal w + mom' bit for bit, and the bf16 shadow must equal the rounding of the kernel's own fp32 w'
-- in the float4 body and in the n & 3 tail.  Each buffer carries a guard region past n in the same allocation that
must come back untouched.  n covers the tail-only sizes 1 - 3, exactly one vector, one vector + tail, a ragged mid size,
a power of two, and a size above 132 * 8 * 256 vectors so the grid-stride loop makes a second trip."""
import pytest

pytestmark = pytest.mark.gpu

E32 = 2.0 ** -23
GUARD = 64
SIZES = [1, 2, 3, 4, 5, 1001, 4096, 1000003, 132 * 8 * 256 * 4 + 4099]


def _buffers(n, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    full = [torch.randn(n + GUARD, generator=g, device="cuda") for _ in range(3)]
    full[2] *= 0.1                                             # gradients
    return full, [t[:n] for t in full]


def _reference(w0, m0, g, lr, wd, momentum, rescale):
    """float64 update from fp32 inputs and the kernel's fp32 scalar products -> (mom', bound on mom')"""
    import torch
    f = lambda v: torch.tensor(v, dtype=torch.float32)
    lrwd, lrrs = float(f(lr) * f(wd)), float(f(lr) * f(rescale))
    t1, t2, t3 = float(f(momentum)) * m0.double(), lrwd * w0.double(), lrrs * g.double()
    return t1 - t2 - t3, 2 * E32 * (t1.abs() + t2.abs() + t3.abs()) + 2.0 ** -149


def _check(w, mom, g, w0, m0, lr, wd, momentum, rescale, full, full0, n, w16=None, w16_full=None):
    import torch
    ref, bound = _reference(w0, m0, g, lr, wd, momentum, rescale)
    err = (mom.double() - ref).abs()
    assert bool((err <= bound).all()), "mom: worst excess %.3e at n = %d" % (float((err - bound).max()), n)
    assert torch.equal(w, w0 + mom), "w' must be the single fp32 sum w + mom'"
    for t, t0 in zip(full, full0):
        assert torch.equal(t[n:], t0[n:]), "memory past n was written"
    assert torch.equal(full[2], full0[2]), "the gradient was modified"
    if w16 is not None:
        assert torch.equal(w16, w.bfloat16()), "bf16 shadow != rounding of the updated fp32 weights"
        assert bool((w16_full[n:] == -7.0).all()), "bf16 shadow written past n"
    return float((err / bound).max())


@pytest.mark.parametrize("momentum", [0.0, 0.9])
@pytest.mark.parametrize("n", SIZES)
def test_sgd_mom(n, momentum):
    import torch
    from sniper_b200 import ops
    full, (w, mom, g) = _buffers(n, 11 + n)
    full0 = [t.clone() for t in full]
    lr, wd, rescale = 0.0123, 1e-4, 0.37
    ops.sgd_mom(w, mom, g, lr=lr, wd=wd, momentum=momentum, rescale=rescale)
    _check(w, mom, g, full0[0][:n], full0[1][:n], lr, wd, momentum, rescale, full, full0, n)


@pytest.mark.parametrize("shadow", [False, True])
@pytest.mark.parametrize("momentum", [0.0, 0.9])
@pytest.mark.parametrize("n", SIZES)
def test_sgd_mom_dev(n, momentum, shadow):
    """lr / wd live on the device: a second call after rewriting `hyper` in place (what a captured update graph relies
    on) must use the new values without anything being re-created."""
    import torch
    from sniper_b200 import ops
    full, (w, mom, g) = _buffers(n, 23 + n)
    w16_full = torch.full((n + GUARD,), -7.0, device="cuda", dtype=torch.bfloat16) if shadow else None
    w16 = w16_full[:n] if shadow else None
    hyper = torch.tensor([0.02, 5e-4], device="cuda")
    lr_mult, wd_mult, rescale = 0.01, 0.5, 1.0 / 16
    f = lambda v: float(torch.tensor(v, dtype=torch.float32))
    for step, (lr0, wd0) in enumerate([(0.02, 5e-4), (0.002, 1e-4)]):
        hyper.copy_(torch.tensor([lr0, wd0]))                               # same device buffer, new schedule values
        full0 = [t.clone() for t in full]
        ops.sgd_mom_dev(w, mom, g, hyper, lr_mult, wd_mult, momentum, rescale, w_bf16=w16)
        lr = f(f(lr0) * f(lr_mult))
        wd = f(f(wd0) * f(wd_mult))
        _check(w, mom, g, full0[0][:n], full0[1][:n], lr, wd, momentum, rescale, full, full0, n, w16, w16_full)
    assert torch.equal(hyper, torch.tensor([0.002, 1e-4], device="cuda")), "hyper is read-only for the kernel"


def test_group_multipliers_zero():
    """lr_mult = 0 freezes a group (mom' = momentum * mom exactly, w' = w + mom'); wd_mult = 0 drops the decay term."""
    import torch
    from sniper_b200 import ops
    n = 1001
    full, (w, mom, g) = _buffers(n, 5)
    w0, m0 = w.clone(), mom.clone()
    hyper = torch.tensor([0.1, 1e-2], device="cuda")
    ops.sgd_mom_dev(w, mom, g, hyper, 0.0, 1.0, 0.5, 1.0)
    assert torch.equal(mom, m0 * 0.5) and torch.equal(w, w0 + mom)
    w0, m0 = w.clone(), mom.clone()
    ops.sgd_mom_dev(w, mom, g, hyper, 1.0, 0.0, 0.0, 1.0)
    ref = -(torch.tensor(0.1) * torch.tensor(1.0)).item() * g.double()
    assert bool(((mom.double() - ref).abs() <= E32 * ref.abs() + 2.0 ** -149).all()) and torch.equal(w, w0 + mom)
