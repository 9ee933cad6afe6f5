"""The depthwise 3x3 forward and data gradient (sniper_depthwise3x3_fwd / _dgrad) and the first-layer im2col
(sniper_im2col3x3s2_nchw) on the device against float64, on every launch path.

Shapes: the 17 depthwise layers of a MobileNetV2 training step (B = 40 on 512 x 512 chips, channels padded to 64 as
the network stores them); the same layers at both orientations of the canvas of every shipped TEST scale
(`iterator.default_config(network="mobilenetv2").TEST`, canvases `tester._canvas_size(h, w, 32)`) with that scale's
batch; ragged maps around the tiles (TH x TW = 8 x 32 at stride 1, 4 x 16 at stride 2) and the register kernels'
strips (PW = 4 / 2), odd and even sizes at stride 2 (the a1 / b1 edges of dgrad_s2), channel counts on the register
path (C % 64 != 0) and on the tiled path with several 64-channel chunks.

Launch paths: bf16 with C % 64 == 0, a pixel stride ld % 8 == 0 and a 16-byte aligned input runs the shared-memory
tiled kernel (forward, stride-1 data gradient), everything else the register-window kernel; the stride-2 data gradient
has its own kernel.  Each case names its path by that rule, `test_launch_path_follows_the_rule` checks the rule against
the kernel names a profiler sees, and every tiled case is rerun on the register path (the same values in a slice with
ld = C + 4, and in a slice big[..., 4:4 + C] of a wider map, whose base is only 8-byte aligned) and must give the same
bytes: both kernels do the same fmas in the same order.

Error bounds, u = 2^-24, S = sum of |terms| of an output, computed in float64 from the stored inputs (exact):
  forward and stride-1 data gradient: a chain of at most 9 fmaf starting from 0     -> b = 10 u S
  stride-2 data gradient: at most 4 terms, one multiply then fmaf                   -> b =  5 u S
fp32 outputs must satisfy |got - exact| <= b; bf16 outputs are the fp32 result rounded to nearest even, which is
monotone, so RNE8(exact - b) <= got <= RNE8(exact + b) with RNE8 a float64 rounding to 8 significant bits (a cast that
truncated instead fails this).  Every case runs a second time on inputs that make every partial sum exact (x integer in
[-3, 3], w in {-2, -1, -1/2, 0, 1/2, 1, 2}: |sum| <= 54 in steps of 1/2 needs 7 bits), where the output must equal
the float64 result: any wrong tap, flip, border or parity shows bit for bit.

Guards: outputs start as NaN and must be finite in [0, C) afterwards (every element written, also every dx of the
stride-2 gradient); the channels [0, lead) and [lead + C, ld) of sliced outputs and one map row before and after the
output keep their NaN bits; input channels outside [lead, lead + C) are NaN and must not reach any output.  The kernels
use no atomics: two eager launches, and a CUDA-graph replay, give the same bytes.  Seeds come from the crc32 of the
case id, so a failure reproduces; the worst err / bound of each (operation, dtype, path) class is reported at the end."""
import zlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
NAN = float("nan")
DT = {"fp32": torch.float32, "bf16": torch.bfloat16}


def _seed(*key):
    return zlib.crc32(repr(key).encode())


def _unit_shapes(B, H, W):
    """(NB, H, W, C, stride) of the depthwise layer of each inverted-residual unit (model_mnv2.MCfg.bottlenecks) for a
    [B, 3, H, W] input."""
    from sniper_b200 import model_mnv2 as MM
    cfg = MM.MCfg()
    H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1                  # first 3x3 / stride 2 conv
    out, cin = [], cfg.first_c
    for t, c, n, s in cfg.bottlenecks:
        for j in range(n):
            e = int(round((cin if j == 0 else c) * t))
            st = s if j == 0 else 1
            out.append((B, H, W, MM.pad64(e), st))
            H, W = (H - 1) // st + 1, (W - 1) // st + 1
        cin = c
    return out


def _test_canvases():
    """(batch, canvas h, canvas w) of both orientations of every TEST scale of the MobileNetV2 config."""
    from sniper_b200 import iterator, tester
    cfg = iterator.default_config(network="mobilenetv2")
    out = []
    for (s0, s1), b in zip(cfg.TEST.SCALES, cfg.TEST.BATCH_IMAGES):
        out.append((b, ) + tester._canvas_size(s0, s1, 32))           # horizontal images
        out.append((b, ) + tester._canvas_size(s1, s0, 32))           # vertical images
    return out


TRAIN = [("train%02d" % i, ) + u + ("dense", ) for i, u in enumerate(_unit_shapes(40, 512, 512))]
assert len(TRAIN) == 17
INFER = [("test%dx%d_u%02d" % (h, w, i), ) + u + ("dense", )
         for b, h, w in _test_canvases() for i, u in enumerate(_unit_shapes(b, h, w))]
# (NB, H, W, C, stride, layout): layout "dense" (ld = C), "ld4" (a slice with ld = C + 4), "off4" (big[..., 4:4 + C]
# of a map with ld = C + 64: the base is 16-byte aligned in fp32, only 8-byte aligned in bf16)
RAGGED = [
    (1, 1, 1, 64, 1, "dense"), (1, 1, 1, 64, 2, "dense"), (1, 1, 1, 4, 1, "dense"), (2, 1, 37, 64, 1, "dense"),
    (2, 1, 37, 192, 2, "dense"), (2, 29, 1, 64, 1, "dense"), (2, 29, 1, 64, 2, "dense"),
    (2, 9, 2, 64, 1, "dense"), (2, 9, 3, 64, 2, "dense"), (2, 9, 5, 64, 1, "dense"), (2, 9, 31, 64, 2, "dense"),
    (2, 9, 33, 64, 1, "dense"), (2, 9, 63, 64, 2, "dense"), (2, 9, 65, 64, 1, "dense"), (2, 8, 65, 64, 2, "dense"),
    (2, 7, 40, 192, 1, "dense"), (2, 9, 40, 192, 2, "dense"), (2, 15, 40, 192, 1, "dense"), (2, 17, 40, 192, 2, "dense"),
    (1, 8, 10, 64, 2, "dense"), (1, 9, 11, 64, 2, "dense"), (1, 8, 11, 64, 2, "dense"), (1, 9, 10, 64, 2, "dense"),
    (2, 17, 33, 4, 1, "dense"), (2, 15, 31, 8, 2, "dense"), (2, 9, 65, 60, 1, "dense"), (1, 33, 17, 60, 2, "dense"),
    (1, 20, 36, 576, 2, "dense"), (2, 10, 14, 960, 1, "dense"), (1, 19, 23, 960, 2, "dense"),
    (2, 16, 16, 192, 1, "dense"), (1, 13, 70, 576, 1, "dense"),
    (2, 17, 33, 64, 1, "ld4"), (2, 17, 33, 64, 2, "ld4"), (2, 15, 31, 60, 2, "ld4"), (1, 9, 65, 192, 1, "ld4"),
    (2, 32, 48, 64, 1, "off4"), (2, 17, 33, 64, 2, "off4"), (1, 9, 65, 192, 1, "off4"), (1, 7, 9, 8, 1, "off4"),
    (1, 11, 37, 576, 2, "off4"),
]
CASES = TRAIN + INFER + [("ragged%02d" % i, ) + r for i, r in enumerate(RAGGED)]

WORST = {}          # (operation, dtype, path) -> (worst err / bound, bound-checked launches, exact-mode launches)


@pytest.fixture(scope="module", autouse=True)
def _report():
    """Prints the worst err / bound of each class when the module is done (shown with -s or -rP)."""
    yield
    print("\ndepthwise fwd / dgrad vs float64: worst err / bound per class")
    for k in sorted(WORST):
        r, n, ne = WORST[k]
        print("  %-9s %s %-8s  %.3g  (%d bound-checked launches, %d exact-mode launches value-equal)" % (k + (r, n, ne)))


def _record(key, ratio, exact_mode):
    r, n, ne = WORST.get(key, (0.0, 0, 0))
    WORST[key] = (max(r, ratio), n + (not exact_mode), ne + exact_mode)


def _layout(C, layout):
    """(lead, ld): the view is channels [lead, lead + C) of pixels ld elements apart."""
    return {"dense": (0, C), "ld4": (0, C + 4), "off4": (4, C + 64)}[layout]


def _path(op, stride, x, C):
    """The kernel the entry point picks for input map x (the use_tiled rule of depthwise.cu)."""
    if op == "dgrad" and stride == 2:
        return "s2"
    tiled = x.dtype == torch.bfloat16 and C % 64 == 0 and x.stride(2) % 8 == 0 and x.data_ptr() % 16 == 0
    return "tiled" if tiled else "register"


def _map(vals, layout):
    """vals [N,h,w,C] placed in a NaN-filled map with the given layout."""
    N, h, w, C = vals.shape
    lead, ld = _layout(C, layout)
    buf = torch.full((N, h, w, ld), NAN, dtype=vals.dtype, device=DEV)
    v = buf[..., lead:lead + C]
    v.copy_(vals)
    return v


def _out(shape, dt, layout):
    """A NaN-filled output view with the given layout, one map row of guard before and after; (buffer, view)."""
    N, h, w, C = shape
    lead, ld = _layout(C, layout)
    buf = torch.full((N * h + 2, w, ld), NAN, dtype=dt, device=DEV)
    return buf, buf[1:N * h + 1].view(N, h, w, ld)[..., lead:lead + C]


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def _check_out(buf, view, shape, layout):
    N, h, w, C = shape
    lead, ld = _layout(C, layout)
    assert torch.isfinite(view).all(), "an output element was not written (or is not finite)"
    rest = buf.clone()
    rest[1:N * h + 1].view(N, h, w, ld)[..., lead:lead + C] = NAN
    assert torch.equal(_bits(rest), _bits(torch.full_like(buf, NAN))), "wrote outside the output view"


def _launch(op, inp, w, stride, H, W, out):
    from sniper_b200 import ops
    if op == "fwd":
        ops.depthwise3x3(inp, w, stride, out=out)
    else:
        ops.depthwise3x3_dgrad(inp, w, (H, W), stride, out=out)


def _run(op, inp, w, stride, H, W, out_shape, layout):
    buf, view = _out(out_shape, inp.dtype, layout)
    _launch(op, inp, w, stride, H, W, view)
    torch.cuda.synchronize()
    _check_out(buf, view, out_shape, layout)
    return view


def _ref(op, v, w, stride, H, W):
    """float64 result and sum of |terms| of the forward (v = x) or the data gradient (v = dy); v [N,h,w,C] and w [9,C]
    float64.  Forward and stride-1 gradient: shifted slices of the zero-padded map; stride-2 gradient: each dy * w[t]
    scattered to dx[2 a + kh - 1, 2 b + kw - 1] (the transposed correlation)."""
    N, _, _, C = v.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    if op == "dgrad" and stride == 2:
        acc = torch.zeros(N, H + 2, W + 2, C, dtype=torch.float64, device=DEV)
        mag = torch.zeros_like(acc)
        for kh in range(3):
            for kw in range(3):
                t = v * w[kh * 3 + kw]
                acc[:, kh:kh + 2 * (Ho - 1) + 1:2, kw:kw + 2 * (Wo - 1) + 1:2] += t
                mag[:, kh:kh + 2 * (Ho - 1) + 1:2, kw:kw + 2 * (Wo - 1) + 1:2] += t.abs_()
                del t
        return acc[:, 1:H + 1, 1:W + 1], mag[:, 1:H + 1, 1:W + 1]
    vp = F.pad(v, (0, 0, 1, 1, 1, 1))
    oh, ow = (Ho, Wo) if op == "fwd" else (H, W)
    acc = torch.zeros(N, oh, ow, C, dtype=torch.float64, device=DEV)
    mag = torch.zeros_like(acc)
    for kh in range(3):
        for kw in range(3):
            if op == "fwd":       # y[ho, wo] += x[ho S + kh - 1, wo S + kw - 1] w[kh, kw]
                vs = vp[:, kh:kh + (Ho - 1) * stride + 1:stride, kw:kw + (Wo - 1) * stride + 1:stride]
            else:                 # dx[h, w] += dy[h + 1 - kh, w + 1 - kw] w[kh, kw]
                vs = vp[:, 2 - kh:2 - kh + H, 2 - kw:2 - kw + W]
            t = vs * w[kh * 3 + kw]
            acc += t
            mag += t.abs_()
            del t
    return acc, mag


def _pow2(k):
    """2.0 ** k for an integer tensor k in the normal float64 range, built from its bits (exact)."""
    return ((k.to(torch.int64) + 1023) << 52).view(torch.float64)


def _rne8(v):
    """float64 v rounded to 8 significant bits, ties to even (bf16's significand; no double rounding).  v = m 2^e with
    0.5 <= |m| < 1: m * 256 is exact and torch.round rounds half to even."""
    m, e = torch.frexp(v)
    return torch.round(m * 256.0) * _pow2(e - 8)


def _bf16_err(g, exact):
    """Distance from exact to the reals that round to the bf16 value g (0 when exact itself rounds to g): the least
    fp32 accumulation error that explains g.  |g| = m 2^e rounds from [|g| - ulp_below / 2, |g| + 2^(e-8) / 2], with
    ulp_below = 2^(e-9) when |g| is a power of two."""
    # g == 0 is taken as the point 0: the reals that round to a bf16 zero lie within 2^-134 of it, far below any bound
    m, e = torch.frexp(g.abs())
    up = _pow2(e - 9)
    dn = torch.where(m == 0.5, _pow2(e - 10), up)
    a_lo, a_hi = g.abs() - dn, g.abs() + up
    lo = torch.where(g > 0, a_lo, torch.where(g < 0, -a_hi, g))
    hi = torch.where(g > 0, a_hi, torch.where(g < 0, -a_lo, g))
    return torch.clamp(torch.maximum(lo - exact, exact - hi), min=0.0)


def test_rne8_is_the_fp32_to_bf16_cast():
    g = torch.Generator(device=DEV)
    g.manual_seed(_seed("rne8"))
    r = torch.randn(1 << 20, device=DEV, generator=g) * torch.exp2(torch.randint(-40, 40, (1 << 20, ), device=DEV,
                                                                                    generator=g).float())
    k = torch.randint(128, 256, (4096, ), device=DEV, generator=g) * 2 + 1          # 9 significant bits, last one set:
    ties = k.float() * torch.exp2(torch.randint(-20, 20, (4096, ), device=DEV, generator=g).float())   # halfway cases
    r = torch.cat([r, ties, -ties, torch.zeros(1, device=DEV)])
    assert torch.equal(_rne8(r.double()), r.to(torch.bfloat16).double())


def _check_bound(got, exact, mag, nterms, what):
    """got within the rounding bound of exact; returns the worst err / bound (bf16: the least fp32 error that explains
    the stored value, over b)."""
    b = (nterms + 1) * U * mag
    g = got.double()
    if got.dtype == torch.float32:
        err = (g - exact).abs()
        ok = err <= b
    else:
        ok = (_rne8(exact - b) <= g) & (g <= _rne8(exact + b))
        err = _bf16_err(g, exact)
    if not ok.all():
        i = tuple((~ok).nonzero()[0].tolist())
        raise AssertionError("%s: at %s got %r, exact %r, bound %r" % (what, list(i), g[i].item(), exact[i].item(),
                                                                     b[i].item()))
    ratio = torch.where(err > 0, err / b, torch.zeros_like(err))
    return ratio.max().item()


def _inputs(shape, C, dt, exact_mode, g):
    if exact_mode:
        v = torch.randint(-3, 4, shape, device=DEV, generator=g).to(dt)
        vals = torch.tensor([-2.0, -1.0, -0.5, 0.0, 0.5, 1.0, 2.0], device=DEV)
        w = vals[torch.randint(0, 7, (9, C), device=DEV, generator=g)]
    else:
        v = torch.randn(shape, device=DEV, generator=g).to(dt)
        w = torch.randn(9, C, device=DEV, generator=g)
    return v, w


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fwd_and_dgrad_match_float64(case, dtype):
    name, (NB, H, W, C, stride, layout) = case[0], case[1:]
    dt = DT[dtype]
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    for op in ("fwd", "dgrad"):
        in_shape, out_shape = ((NB, H, W, C), (NB, Ho, Wo, C)) if op == "fwd" else ((NB, Ho, Wo, C), (NB, H, W, C))
        nterms = 4 if op == "dgrad" and stride == 2 else 9
        for exact_mode in (False, True):
            what = "%s %s %s %s" % (name, dtype, op, "exact" if exact_mode else "random")
            g = torch.Generator(device=DEV)
            g.manual_seed(_seed(name, dtype, op, exact_mode))
            vals, w = _inputs(in_shape, C, dt, exact_mode, g)
            inp = _map(vals, layout)
            path = _path(op, stride, inp, C)
            if dtype == "fp32" or C % 64:
                assert path in ("register", "s2"), what
            elif layout == "dense":
                assert path in ("tiled", "s2"), what
            got = _run(op, inp, w, stride, H, W, out_shape, layout)
            exact, mag = _ref(op, vals.double(), w.double(), stride, H, W)
            if exact_mode:
                assert torch.equal(got.double(), exact), what + ": not value-equal to the exact result"
                ratio = 0.0
            else:
                ratio = _check_bound(got, exact, mag, nterms, what)
            del exact, mag
            key = ("fwd" if op == "fwd" else "dgrad-s%d" % stride, dtype, path)
            _record(key, ratio, exact_mode)
            if exact_mode:
                continue
            print("%s: %s path, worst err/bound %.3g" % (what, path, ratio))
            # a second eager launch: the same bytes
            again = _run(op, inp, w, stride, H, W, out_shape, layout)
            assert torch.equal(_bits(again), _bits(got)), what + ": two eager launches differ"
            del again
            if path == "tiled":
                # the same values through the register kernel: a slice with ld % 8 != 0, and one with an 8-byte base
                for alt in ("ld4", "off4"):
                    ainp = _map(vals, alt)
                    assert _path(op, stride, ainp, C) == "register", (what, alt)
                    agot = _run(op, ainp, w, stride, H, W, out_shape, alt)
                    assert torch.equal(_bits(agot), _bits(got)), "%s: register path (%s) differs from tiled" % (what, alt)
                    _record(key[:2] + ("register", ), ratio, False)
                    del ainp, agot
            del got, inp, vals


# the kernel each configuration must reach: (op, dtype, C, stride, layout) -> fragments of its demangled name
PATHS = [
    ("fwd", "fp32", 64, 1, "dense", ("dw_fwd_kernel<float", "false>")),
    ("fwd", "fp32", 64, 2, "dense", ("dw_fwd_kernel<float", "false>")),
    ("fwd", "bf16", 64, 1, "dense", ("dw_fwd_tiled_kernel<", "false>")),
    ("fwd", "bf16", 192, 2, "dense", ("dw_fwd_tiled_kernel<", "false>")),
    ("fwd", "bf16", 64, 1, "ld4", ("dw_fwd_kernel<__nv_bfloat16", "false>")),
    ("fwd", "bf16", 64, 2, "off4", ("dw_fwd_kernel<__nv_bfloat16", "false>")),
    ("fwd", "bf16", 60, 1, "dense", ("dw_fwd_kernel<__nv_bfloat16", "false>")),
    ("dgrad", "fp32", 64, 1, "dense", ("dw_fwd_kernel<float", "true>")),
    ("dgrad", "bf16", 64, 1, "dense", ("dw_fwd_tiled_kernel<", "true>")),
    ("dgrad", "bf16", 64, 1, "off4", ("dw_fwd_kernel<__nv_bfloat16", "true>")),
    ("dgrad", "bf16", 8, 1, "dense", ("dw_fwd_kernel<__nv_bfloat16", "true>")),
    ("dgrad", "fp32", 64, 2, "dense", ("dw_dgrad_s2_kernel<float>", )),
    ("dgrad", "bf16", 64, 2, "dense", ("dw_dgrad_s2_kernel<__nv_bfloat16>", )),
]


@pytest.mark.parametrize("op,dtype,C,stride,layout,kernel", PATHS, ids=["-".join(map(str, p[:5])) for p in PATHS])
def test_launch_path_follows_the_rule(op, dtype, C, stride, layout, kernel):
    """The rule _path restates (and every case above relies on) against the kernel a profiler sees launched."""
    from torch.profiler import ProfilerActivity, profile
    NB, H, W = 2, 12, 20
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    in_shape, out_shape = ((NB, H, W, C), (NB, Ho, Wo, C)) if op == "fwd" else ((NB, Ho, Wo, C), (NB, H, W, C))
    g = torch.Generator(device=DEV)
    g.manual_seed(_seed("path", op, dtype, C, stride, layout))
    vals, w = _inputs(in_shape, C, DT[dtype], False, g)
    inp = _map(vals, layout)
    want = {"tiled": "dw_fwd_tiled_kernel<", "register": "dw_fwd_kernel<", "s2": "dw_dgrad_s2_kernel<"}
    assert kernel[0].startswith(want[_path(op, stride, inp, C)])
    buf, view = _out(out_shape, inp.dtype, layout)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _launch(op, inp, w, stride, H, W, view)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "dw_" in e.name]
    assert len(names) == 1 and all(f in names[0] for f in kernel), names
    _check_out(buf, view, out_shape, layout)


@pytest.mark.parametrize("case", [("tiled", "fwd", "bf16", (4, 64, 96, 192, 1), "dense"),
                                  ("register", "dgrad", "bf16", (4, 64, 96, 192, 1), "ld4"),
                                  ("s2", "dgrad", "fp32", (4, 63, 95, 64, 2), "dense")], ids=lambda c: c[0])
def test_graph_replay_is_byte_identical_to_eager(case):
    name, op, dtype, (NB, H, W, C, stride), layout = case
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    in_shape, out_shape = ((NB, H, W, C), (NB, Ho, Wo, C)) if op == "fwd" else ((NB, Ho, Wo, C), (NB, H, W, C))
    g = torch.Generator(device=DEV)
    g.manual_seed(_seed("graph", name))
    vals, w = _inputs(in_shape, C, DT[dtype], False, g)
    inp = _map(vals, layout)
    assert _path(op, stride, inp, C) == name
    eager = _run(op, inp, w, stride, H, W, out_shape, layout)
    buf, view = _out(out_shape, inp.dtype, layout)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _launch(op, inp, w, stride, H, W, view)
    for i in range(2):
        view.fill_(NAN)
        graph.replay()
        torch.cuda.synchronize()
        _check_out(buf, view, out_shape, layout)
        assert torch.equal(_bits(view), _bits(eager)), "replay %d differs from eager" % i


# ---- first-layer im2col: [N,3,H,W] fp32 -> [N,Ho,Wo,Kp] rows of 3x3 / stride-2 patches in (kh, kw, ci) order
IM2COL = [("train", 40, 512, 512, 64, "fp32"), ("train", 40, 512, 512, 64, "bf16"), ("odd", 2, 511, 385, 64, "fp32"),
          ("odd", 2, 511, 385, 64, "bf16"), ("1x1", 1, 1, 1, 64, "fp32"), ("1x1", 1, 1, 1, 64, "bf16"),
          ("2x3", 2, 2, 3, 64, "fp32"), ("2x3", 2, 2, 3, 64, "bf16"), ("kp28", 3, 37, 23, 28, "fp32"),
          ("kp32", 3, 37, 23, 32, "fp32"), ("kp28", 3, 37, 23, 28, "bf16")]


@pytest.mark.parametrize("name,NB,H,W,Kp,dtype", IM2COL, ids=["%s-%s" % (c[0], c[5]) for c in IM2COL])
def test_im2col3x3s2_matches_unfold_bit_for_bit(name, NB, H, W, Kp, dtype):
    from sniper_b200 import ops
    dt = DT[dtype]
    g = torch.Generator(device=DEV)
    g.manual_seed(_seed("im2col", name, dtype))
    x = torch.randn(NB, 3, H, W, device=DEV, generator=g) * 50
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    u = F.unfold(x, 3, padding=1, stride=2).view(NB, 3, 9, Ho * Wo)         # rows (ci, kh, kw)
    want = torch.zeros(NB, Ho, Wo, Kp, device=DEV)
    want[..., :27] = u.permute(0, 3, 2, 1).reshape(NB, Ho, Wo, 27)           # columns (kh, kw, ci), zeros to Kp
    want = want.to(dt)
    buf, col = _out((NB, Ho, Wo, Kp), dt, "dense")
    ops.im2col3x3s2(x, Kp, dtype=dt, out=col)
    torch.cuda.synchronize()
    _check_out(buf, col, (NB, Ho, Wo, Kp), "dense")
    assert torch.equal(_bits(col), _bits(want))
