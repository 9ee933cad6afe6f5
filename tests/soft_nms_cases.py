"""Seeded soft-NMS problems for the batched device soft-NMS (ops.soft_nms_batched), shared by
tests/test_soft_nms_cases_cpu.py (the restatement, the host port and the reference's Cython agree on them, and the
builders produce what they claim) and tests/test_soft_nms_exact_gpu.py (the CUDA kernel against the host port).

A problem is one (image, class) of `inference.aggregate`: float32 rows [n,5] = (x1, y1, x2, y2, score).  The score
regimes are where the order of the reference loop (lib/nms/cpu_nms.pyx:17-110) is decided by its swaps: exact ties
(quantised scores, a saturated softmax at 1.0f, duplicated rows from overlapping chips), rows at or below the score
threshold, and rounds that remove many rows at once.  Sizes straddle the kernel's 256-thread block stride."""
import functools
import importlib
import os
import sys

import numpy as np
import pytest

W, H = 1333, 800
THRESHOLD = np.float32(0.001)
ONE_BELOW_ONE = np.float32(np.nextafter(np.float32(1.0), np.float32(0.0)))    # 0.99999994f
# (method, sigma, Nt): 1 linear, 2 Gaussian as `inference.aggregate` calls it, 3 hard NMS
METHODS = ((1, 0.5, 0.3), (2, 0.55, 0.3), (3, 0.5, 0.3))
REGIMES = ("tie_free", "q8", "q64", "q1000", "saturated", "all_equal", "duplicates", "low_scores", "disjoint",
           "identical_boxes", "heavy_decay")
TIE_REGIMES = tuple(r for r in REGIMES if r != "tie_free")
SIZES = (2, 255, 256, 257, 511)          # around the 256-thread block stride of the kernel
AGGREGATED_ROWS = 4000                   # one class of an image after three scales of chips


def _clustered_boxes(rng, n, spread=15.0):
    """Detections of a few objects: log-uniform sizes in [8, 400] px, aspect in [0.5, 2], centres around ~n/12
    object centres, clipped to the image."""
    s = np.exp(rng.uniform(np.log(8), np.log(400), n))
    ar = np.exp(rng.uniform(np.log(0.5), np.log(2.0), n))
    w, h = s * np.sqrt(ar), s / np.sqrt(ar)
    k = max(1, n // 12)
    cx = rng.uniform(0, W, k)[rng.randint(0, k, n)] + rng.randn(n) * spread
    cy = rng.uniform(0, H, k)[rng.randint(0, k, n)] + rng.randn(n) * spread
    return np.stack([np.clip(cx - w / 2, 0, W - 1), np.clip(cy - h / 2, 0, H - 1), np.clip(cx + w / 2, 0, W - 1),
                     np.clip(cy + h / 2, 0, H - 1)], 1).astype(np.float32)


def _tie_free(rng, n, lo=0.001, hi=0.999):
    """n distinct scores, log-uniform in (lo, hi) as detection scores are: most rows are low, and the Gaussian decays
    the lowest below the threshold."""
    u = (rng.permutation(n) + 1.0) / (n + 1.0)
    return np.exp(np.log(lo) + (np.log(hi) - np.log(lo)) * u).astype(np.float32)


def _quantised(rng, n, q):
    """Scores k / q, k in 1..q log-uniformly, plus 20 % of the rows at exactly 1.0."""
    k = np.maximum(1, np.round(q * np.exp(rng.uniform(np.log(1.0 / q), 0.0, n))))
    s = (k / float(q)).astype(np.float32)
    s[rng.permutation(n)[:n // 5]] = 1.0
    return s


def _saturated(rng, n):
    """A saturated softmax: continuous scores, 10-30 % of the rows at exactly 1.0f and 5 % at the float below it."""
    s = _tie_free(rng, n)
    idx = rng.permutation(n)
    m = int(round(n * rng.uniform(0.1, 0.3)))
    s[idx[:m]] = 1.0
    s[idx[m:m + n // 20]] = ONE_BELOW_ONE
    return s


def _grid_boxes(n, step=30.0, size=20.0):
    """n boxes on a grid, `step` apart and `size` wide: with the +1 extents no two of them overlap."""
    cols = int(np.ceil(np.sqrt(n)))
    r, c = np.divmod(np.arange(n), cols)
    x1, y1 = c * step + 0.25, r * step + 0.5
    return np.stack([x1, y1, x1 + size, y1 + size], 1).astype(np.float32)


def _rows(regime, rng, n):
    """[n,5] float32 rows of one regime."""
    if regime == "tie_free":
        return np.concatenate([_clustered_boxes(rng, n), _tie_free(rng, n)[:, None]], 1)
    if regime in ("q8", "q64", "q1000"):
        return np.concatenate([_clustered_boxes(rng, n), _quantised(rng, n, int(regime[1:]))[:, None]], 1)
    if regime == "saturated":
        return np.concatenate([_clustered_boxes(rng, n), _saturated(rng, n)[:, None]], 1)
    if regime == "all_equal":
        return np.concatenate([_clustered_boxes(rng, n), np.full((n, 1), 0.75, np.float32)], 1)
    if regime == "duplicates":
        # overlapping chips report the same detection again: three chips, each a random subset of the objects' rows in
        # the same order, so exact copies (same box, same score) sit far apart in the problem
        m = max(1, (n + 1) // 2)
        base = np.concatenate([_clustered_boxes(rng, m), _saturated(rng, m)[:, None]], 1)
        chips = [base[np.sort(rng.permutation(m)[:max(1, (n + 2) // 3)])] for _ in range(3)]
        out = np.concatenate(chips, 0)[:n]
        if len(out) < n:
            out = np.concatenate([out, base[:n - len(out)]], 0)
        return out
    if regime == "low_scores":
        # rows at or below the score threshold: below it, exactly 0.0 and exactly float32(0.001)
        s = _quantised(rng, n, 64)
        idx = rng.permutation(n)
        k = max(1, n // 10)
        s[idx[:k]] = 0.0
        s[idx[k:2 * k]] = THRESHOLD
        s[idx[2 * k:3 * k]] = (rng.randint(1, 1000, len(idx[2 * k:3 * k])) * 1e-6).astype(np.float32)
        return np.concatenate([_clustered_boxes(rng, n), s[:, None]], 1)
    if regime == "disjoint":
        # no two boxes overlap: nothing decays, the output is the swap order of the takes alone
        return np.concatenate([_grid_boxes(n)[rng.permutation(n)], _quantised(rng, n, 8)[:, None]], 1)
    if regime == "identical_boxes":
        # a handful of boxes, each repeated many times: hard NMS keeps one of each, the Gaussian only decays
        groups = _clustered_boxes(rng, 4, spread=0.0)
        b = groups[rng.randint(0, len(groups), n)]
        return np.concatenate([b, _quantised(rng, n, 8)[:, None]], 1)
    if regime == "heavy_decay":
        # tight clusters of low scores under a few confident rows: the first takes push many rows below 0.001 in one
        # round, so the reference's swap-with-last cascades
        c = _clustered_boxes(rng, max(1, n // 64), spread=0.0)
        b = c[rng.randint(0, len(c), n)] + rng.uniform(-1.5, 1.5, (n, 4)).astype(np.float32)
        s = (rng.randint(1, 9, n) / 4000.0).astype(np.float32)
        s[rng.permutation(n)[:max(1, n // 50)]] = 1.0
        return np.concatenate([b, s[:, None]], 1)
    raise ValueError(regime)


def _aggregated(rng, n):
    """One class of one image after three scales: the same objects seen at each scale and, within a scale, by
    overlapping chips (exact duplicate rows), scores of a saturated softmax.  Rows stacked scale by scale, chip by
    chip, as `inference.aggregate` stacks them."""
    objs = _clustered_boxes(rng, 40)
    parts = []
    while sum(len(p) for p in parts) < n:
        for _scale in range(3):
            m = 200
            o = objs[rng.randint(0, len(objs), m)]
            b = np.clip(o + rng.randn(m, 4).astype(np.float32) * 3.0, 0, W - 1)
            b = np.concatenate([np.minimum(b[:, :2], b[:, 2:]), np.maximum(b[:, :2], b[:, 2:])], 1)
            rows = np.concatenate([b, _saturated(rng, m)[:, None]], 1).astype(np.float32)
            dup = rows[rng.permutation(m)[:m // 4]]                   # seen again by the next chip
            parts += [rows, dup]
    return np.concatenate(parts, 0)[:n].astype(np.float32)


def _cases():
    out = [("empty", "tie_free", 0, 0), ("single", "saturated", 1, 1), ("single_zero", "low_scores", 1, 2)]
    k = 3
    for regime in REGIMES:
        for n in SIZES:
            out.append(("%s-%d" % (regime, n), regime, n, k))
            k += 1
    out.append(("aggregated-%d" % AGGREGATED_ROWS, "aggregated", AGGREGATED_ROWS, k))
    out.append(("heavy_decay-%d" % AGGREGATED_ROWS, "heavy_decay", AGGREGATED_ROWS, k + 1))
    return out


CASES = _cases()
CASE_NAMES = [c[0] for c in CASES]


@functools.lru_cache(maxsize=None)
def build(name):
    """float32 rows [n,5] of case `name` (read-only)."""
    _, regime, n, seed = next(c for c in CASES if c[0] == name)
    rng = np.random.RandomState(9100 + seed)
    if regime == "aggregated":
        d = _aggregated(rng, n)
    elif name == "single_zero":
        d = np.array([[10.5, 20.25, 60.0, 90.75, 0.0]], np.float32)
    else:
        d = _rows(regime, rng, n)
    d = np.ascontiguousarray(d, dtype=np.float32).reshape(n, 5)
    assert np.all(d[:, 4] >= 0) and np.all(d[:, 2] >= d[:, 0]) and np.all(d[:, 3] >= d[:, 1])
    d.setflags(write=False)
    return d


def regime(name):
    return next(c[1] for c in CASES if c[0] == name)


def host_soft_nms(d, sigma, Nt, method):
    """The host port (bit-identical to the reference's loop) on a copy of d."""
    from sniper_b200 import host
    return host.cpu_soft_nms(d.copy(), sigma=sigma, Nt=Nt, threshold=float(THRESHOLD), method=method) if len(d) else d


def ref_cython():
    """The reference's own Cython cpu_nms module (oracle/_ref, built by build() where the reference tree is), or skip."""
    ref_dir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")
    if ref_dir not in sys.path:
        sys.path.insert(0, ref_dir)
    try:
        return importlib.import_module("ref_cpu_nms")
    except ImportError:
        pytest.skip("oracle/_ref/ref_cpu_nms not built (needs the reference tree and Cython at build time)")


def cython_soft_nms(ref, d, sigma, Nt, method):
    return np.array(ref.cpu_soft_nms(d.copy(), sigma=sigma, Nt=Nt, threshold=float(THRESHOLD), method=method),
                    np.float32).reshape(-1, 5)


def assert_same_output(got, want, method, what):
    """Same rows in the same order; scores equal, or for the Gaussian within 1 ulp / 2e-7 (its weight is a double exp:
    glibc on the host, CUDA libm on the device, np.exp on a float in the Cython)."""
    assert got.shape == want.shape, "%s: %d rows vs %d" % (what, len(got), len(want))
    assert np.array_equal(got[:, :4], want[:, :4]), "%s: rows or order differ" % what
    if method == 2:
        ulp = np.abs(got[:, 4].view(np.int32).astype(np.int64) - want[:, 4].view(np.int32).astype(np.int64))
        assert ulp.max(initial=0) <= 1 and np.abs(got[:, 4] - want[:, 4]).max(initial=0) <= 2e-7, what
    else:
        assert np.array_equal(got[:, 4], want[:, 4]), "%s: scores differ" % what
