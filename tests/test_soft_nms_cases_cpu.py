"""The soft-NMS order on exact score ties, on the CPU: a numpy restatement of the reference loop
(lib/nms/cpu_nms.pyx:17-110) in the order-free form the device kernel (csrc/nms.cu) computes it, with the reference's
positions tracked, against the host port (host.cpu_soft_nms) and the reference's own Cython (oracle/_ref/ref_cpu_nms,
when built) on every case of tests/soft_nms_cases.py.  Also: the rule the kernel used before it tracked positions
(ties to the lowest input row) differs from the reference on the tie cases, and each case has the property its name
claims."""
import numpy as np
import pytest

import soft_nms_cases as C

F32, F64 = np.float32, np.float64


def _decay(d, score, rows, t, sigma, Nt, method, threshold):
    """The reference's decay of `rows` against the taken row t, in its arithmetic (float IoU with the `+ 1` sums in
    double, the Gaussian weight through a double exp).  Returns (overlapping mask, new scores, removed mask)."""
    x1, y1, x2, y2 = (d[rows, c] for c in range(4))
    tx1, ty1, tx2, ty2 = (d[t, c] for c in range(4))
    area = (((x2 - x1).astype(F64) + 1.0) * ((y2 - y1).astype(F64) + 1.0)).astype(F32)
    iw = ((np.minimum(tx2, x2) - np.maximum(tx1, x1)).astype(F64) + 1.0).astype(F32)
    ih = ((np.minimum(ty2, y2) - np.maximum(ty1, y1)).astype(F64) + 1.0).astype(F32)
    hit = (iw > 0) & (ih > 0)
    inter = iw * ih
    tarea = (F64(tx2 - tx1) + 1.0) * (F64(ty2 - ty1) + 1.0)
    ua = ((tarea + area.astype(F64)) - inter.astype(F64)).astype(F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        ov = inter / ua
        if method == 1:
            w = np.where(ov > F32(Nt), (1.0 - ov.astype(F64)).astype(F32), F32(1))
        elif method == 2:
            w = np.exp((-(ov * ov) / F32(sigma)).astype(F64)).astype(F32)
        else:
            w = np.where(ov > F32(Nt), F32(0), F32(1))
    ns = (w.astype(F32) * score[rows]).astype(F32)
    return hit, ns, hit & (ns < F32(threshold))


def soft_nms_spec(dets, sigma, Nt, method, threshold=C.THRESHOLD, track_positions=True, removed_per_round=None):
    """Soft-NMS restated order-free, as the device kernel computes it.  Every remaining row r has a position pos[r]
    (at first its input row) and at[q] is the row at position q; positions i..N-1 hold the remaining rows.  Take i:
    among the remaining rows with the maximal score, the one at the lowest position (the reference's strict `<`
    scan from i); the row at position i moves to the taken row's position.  Decay: every other remaining row once
    (whether a row survives does not depend on its position).  Compaction (the reference's swap-with-last, replayed):
    with M survivors at positions i+1..N-1, survivors below i+1+M stay, the h-th hole of [i+1, i+1+M) counting up
    gets the h-th survivor at >= i+1+M counting down from the end, and N becomes i+1+M.
    track_positions=False: the rule before positions were tracked, ties to the lowest input row.
    Returns the taken rows in order, each with its score when taken (= the reference's returned array)."""
    d = np.array(dets, F32).reshape(-1, 5)
    n = len(d)
    score = d[:, 4].copy()
    pos, at = np.arange(n), np.arange(n)
    N, out = n, []
    for i in range(n):
        if i >= N:
            break
        rem = at[i:N]
        cand = rem[score[rem] == score[rem].max()]
        k = cand[np.argmin(pos[cand])] if track_positions else cand.min()
        p, r = pos[k], at[i]
        at[p], pos[r] = r, p
        at[i], pos[k] = k, i
        out.append(np.append(d[k, :4], score[k]))
        rest = at[i + 1:N].copy()
        hit, ns, dead = _decay(d, score, rest, k, sigma, Nt, method, threshold)
        score[rest[hit]] = ns[hit]
        M = int((~dead).sum())
        holes = np.flatnonzero(dead[:M])
        tail = rest[M:][~dead[M:]][::-1]
        assert len(holes) == len(tail)
        at[i + 1 + holes] = tail
        pos[tail] = i + 1 + holes
        N = i + 1 + M
        if removed_per_round is not None:
            removed_per_round.append(int(dead.sum()))
    return np.array(out, F32).reshape(-1, 5)


@pytest.mark.parametrize("method,sigma,Nt", C.METHODS)
@pytest.mark.parametrize("name", C.CASE_NAMES)
def test_restatement_matches_host_port(name, method, sigma, Nt):
    d = C.build(name)
    C.assert_same_output(soft_nms_spec(d, sigma, Nt, method), C.host_soft_nms(d, sigma, Nt, method), method, name)


@pytest.mark.parametrize("method,sigma,Nt", C.METHODS)
@pytest.mark.parametrize("name", C.CASE_NAMES)
def test_restatement_and_host_port_match_reference_cython(name, method, sigma, Nt):
    ref = C.ref_cython()
    d = C.build(name)
    want = C.cython_soft_nms(ref, d, sigma, Nt, method)
    C.assert_same_output(C.host_soft_nms(d, sigma, Nt, method), want, method, name + ": host port vs Cython")
    C.assert_same_output(soft_nms_spec(d, sigma, Nt, method), want, method, name + ": restatement vs Cython")


# (case, method) pairs of the tie regimes on which ties to the lowest input row give another output than the
# reference: the seeded cases reach 91 of 162 (linear 34, Gaussian 20, hard 37)
OLD_RULE_MIN_FAILURES = 85
OLD_RULE_MIN_FAILURES_PER_METHOD = 15


def test_lowest_row_rule_fails_on_tie_cases():
    """The cases discriminate: breaking ties by the lowest input row (the kernel's rule before it tracked positions)
    changes the output on many tie cases of every method, and on no tie-free case."""
    failed = []
    for name in C.CASE_NAMES:
        d = C.build(name)
        for method, sigma, Nt in C.METHODS:
            new, old = soft_nms_spec(d, sigma, Nt, method), soft_nms_spec(d, sigma, Nt, method, track_positions=False)
            if old.shape != new.shape or not np.array_equal(old, new):
                failed.append((name, method))
    assert not [f for f in failed if C.regime(f[0]) == "tie_free"], failed
    assert len(failed) >= OLD_RULE_MIN_FAILURES, (len(failed), failed)
    for method, _, _ in C.METHODS:
        assert sum(m == method for _, m in failed) >= OLD_RULE_MIN_FAILURES_PER_METHOD, (method, failed)


def _overlap_pairs(b):
    """#(i < j) with iw > 0 and ih > 0 under the reference's +1 extents."""
    iw = np.minimum(b[:, None, 2], b[None, :, 2]) - np.maximum(b[:, None, 0], b[None, :, 0]) + 1
    ih = np.minimum(b[:, None, 3], b[None, :, 3]) - np.maximum(b[:, None, 1], b[None, :, 1]) + 1
    return int(np.triu((iw > 0) & (ih > 0), 1).sum())


@pytest.mark.parametrize("name", C.CASE_NAMES)
def test_case_has_its_property(name):
    d = C.build(name)
    n, s, reg = len(d), d[:, 4], C.regime(name)
    assert d.dtype == np.float32 and d.shape == (n, 5)
    ties = n - len(np.unique(s))
    if reg == "tie_free":
        assert ties == 0
    elif reg in ("q8", "q64", "q1000"):
        q = int(reg[1:])
        assert np.array_equal(s, np.round(s.astype(F64) * q).astype(F32) / F32(q))
        assert (s == 1.0).sum() >= n // 5
        assert n < 3 or ties > 0
    elif reg == "saturated":
        ones = int((s == 1.0).sum())
        assert 0.1 * n - 1 <= ones <= 0.3 * n + 1 and (s == C.ONE_BELOW_ONE).sum() == n // 20
        assert n < 255 or (ones >= 25 and (s == C.ONE_BELOW_ONE).sum() > 0)
        assert len(np.unique(s[(s != 1.0) & (s != C.ONE_BELOW_ONE)])) == ((s != 1.0) & (s != C.ONE_BELOW_ONE)).sum()
    elif reg == "all_equal":
        assert len(np.unique(s)) == 1
    elif reg in ("duplicates", "aggregated"):
        assert n < 3 or len(np.unique(d, axis=0)) < n             # exact copies: same box, same score
        assert n < 255 or (s == 1.0).sum() >= 25
    elif reg == "low_scores":
        assert n < 255 or ((s == 0).any() and (s == C.THRESHOLD).any() and ((s > 0) & (s < C.THRESHOLD)).any())
        assert name != "single_zero" or s[0] == 0
    elif reg == "disjoint":
        assert _overlap_pairs(d) == 0 and (n < 3 or ties > 0)
    elif reg == "identical_boxes":
        assert len(np.unique(d[:, :4], axis=0)) <= 4 and (n < 3 or ties > 0)
    elif reg == "heavy_decay":
        # many rows leave in a single round, for every method
        for method, sigma, Nt in C.METHODS:
            removed = []
            soft_nms_spec(d, sigma, Nt, method, removed_per_round=removed)
            assert n < 255 or max(removed) >= 20, (method, max(removed, default=0))
    else:
        raise AssertionError(reg)


def test_sizes_straddle_the_block_stride():
    sizes = {len(C.build(n)) for n in C.CASE_NAMES}
    assert {0, 1, 2, 255, 256, 257, 511, C.AGGREGATED_ROWS} <= sizes
    for reg in C.REGIMES:
        assert {len(C.build(n)) for n in C.CASE_NAMES if C.regime(n) == reg} >= set(C.SIZES)
