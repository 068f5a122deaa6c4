"""CPU-only: the scan-matcher oracle (oracle/icp_ref.c) under the settings `parse_icp_yaml` accepts besides the shipped
ones, checked against an independent numpy restatement of one iteration (max_iterations = 1):

  * nearest neighbours by float32 brute force (unfused dx*dx + dy*dy), lowest target index on ties, accepted when the
    squared distance is <= maxDist^2;
  * the keep mask of the MaxDist filter (squared, or raw with flags bit 0) and of the trimmed quantile (element
    floor(float(n_finite) * ratio) of the ascending finite distances, the maximum for ratio 1.0);
  * status and inlier count exactly; T within 1e-5 of a float64 closed-form rigid fit of the kept pairs.

Run on dyadic lattices that put source points exactly on the matcher, outlier and quantile edges and on 2- and 4-way
ties (every edge is counted before it is relied on), and on random pairs for every setting of the grid."""
import itertools

import numpy as np
import pytest

from oracle import oracle as orc
from sonar_slam_b200 import synth

F32 = np.float32
ONE = dict(max_iterations=1, smooth_length=0)
MATCHER = [float("inf"), 1e9, 0.3, 10.0]
OUTLIER = [("off", -1.0, 0), ("squared", 2.0, 0), ("raw", 2.0, 1)]
TRIM = [-1.0, 1.0, 0.0, 0.5, 0.95]


def _mat3(a, b):
    """oracle/icp_ref.c mat3_mul in float32: k ascending, one rounding per operation."""
    a, b = a.astype(F32), b.astype(F32)
    c = np.empty((3, 3), F32)
    for i in range(3):
        for j in range(3):
            acc = a[i, 0] * b[0, j]
            acc = acc + a[i, 1] * b[1, j]
            c[i, j] = acc + a[i, 2] * b[2, j]
    return c


def _nn(step, ref, max_d2):
    """float32 brute force: (index or -1, squared distance or inf); argmin keeps the lowest index of equal minima."""
    idx = np.empty(len(step), np.int64)
    d2 = np.empty(len(step), F32)
    for a in range(0, len(step), 512):
        q = step[a:a + 512]
        dx = q[:, None, 0] - ref[None, :, 0]
        dy = q[:, None, 1] - ref[None, :, 1]
        d = dx * dx + dy * dy
        j = np.argmin(d, axis=1)
        idx[a:a + 512], d2[a:a + 512] = j, d[np.arange(len(q)), j]
    ok = d2 <= max_d2
    return np.where(ok, idx, -1), np.where(ok, d2, F32(np.inf))


def restate_one_iteration(src, tgt, guess, prm):
    """(status, inliers, T float64 or None, details) of one ICP iteration under the oracle's parameters `prm`."""
    src, tgt = np.asarray(src, F32), np.asarray(tgt, F32)
    g = np.asarray(guess, F32)
    if len(tgt) == 0:
        return 6, 0, None, {}
    mx = np.cumsum(tgt[:, 0], dtype=F32)[-1] / F32(len(tgt))  # sequential float32 sums, like the oracle
    my = np.cumsum(tgt[:, 1], dtype=F32)[-1] / F32(len(tgt))
    ref = np.c_[tgt[:, 0] - mx, tgt[:, 1] - my]
    T0 = _mat3(np.array([[1, 0, -mx], [0, 1, -my], [0, 0, 1]], F32), g)
    step = np.c_[(T0[0, 0] * src[:, 0] + T0[0, 1] * src[:, 1]) + T0[0, 2],
                 (T0[1, 0] * src[:, 0] + T0[1, 1] * src[:, 1]) + T0[1, 2]].astype(F32)
    max_d2 = F32(prm.matcher_max_dist) * F32(prm.matcher_max_dist)
    match, d2 = _nn(step, ref, max_d2)
    fin = match >= 0
    keep = fin.copy()
    if prm.outlier_max_dist > 0:
        out_d2 = F32(prm.outlier_max_dist) if prm.flags & 1 else F32(prm.outlier_max_dist) * F32(prm.outlier_max_dist)
        keep &= d2 <= out_d2
    limit = None
    if prm.trim_ratio >= 0:
        if not fin.any():
            return 1, 0, None, {}
        s = np.sort(d2[fin])
        limit = s[-1] if F32(prm.trim_ratio) == F32(1.0) else s[int(F32(len(s)) * F32(prm.trim_ratio))]
        keep &= d2 <= limit
    if not keep.any():
        return 2, 0, None, {}
    # float64 closed-form fit of the kept pairs in the caller's frame (the centring cancels in exact arithmetic)
    G = g.astype(np.float64)
    p = src[keep].astype(np.float64) @ G[:2, :2].T + G[:2, 2]
    r = tgt[match[keep]].astype(np.float64)
    mp, mr = p.mean(0), r.mean(0)
    M = (r - mr).T @ (p - mp)
    th = np.arctan2(M[1, 0] - M[0, 1], M[0, 0] + M[1, 1])
    dT = np.eye(3)
    dT[:2, :2] = [[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]
    dT[:2, 2] = mr - dT[:2, :2] @ mp
    return 0, int(keep.sum()), dT @ G, dict(match=match, d2=d2, keep=keep, limit=limit, max_d2=max_d2)


def _check(src, tgt, guess, **kw):
    prm = orc.IcpParams(**{**ONE, **kw})
    st, inl, T, det = restate_one_iteration(src, tgt, guess, prm)
    r = orc.icp(src, tgt, guess, prm)
    assert r["status"] == st, (kw, r["status"], st)
    assert r["inliers"] == inl, (kw, r["inliers"], inl)
    if st == 0:
        assert r["iterations"] == 1
        assert np.abs(r["T"].astype(np.float64) - T).max() < 1e-5, (kw, r["T"], T)
    else:
        assert np.array_equal(r["T"], np.asarray(guess, F32))
    return det


# ------------------------------------------------------------------ knife-edge lattices
def lattice(k, step=1.0):
    """(2k+1)^2 points on a dyadic square lattice centred on 0: every partial float32 sum is exact, so the oracle's
    centring is exact (mean 0) in any summation order."""
    a = np.arange(-k, k + 1, dtype=np.float64) * step
    return np.array(list(itertools.product(a, a)), F32)


def knife_source(k, offsets, rng, n_each=120):
    """n_each points at every offset from a random interior lattice point (offsets in lattice units)."""
    out = []
    for o in offsets:
        c = rng.integers(-k + 2, k - 1, size=(n_each, 2)).astype(np.float64)
        out.append(c + np.asarray(o, np.float64))
    s = np.concatenate(out).astype(F32)
    return s[rng.permutation(len(s))]


def _shuffled(tgt, seed):
    return tgt[np.random.default_rng(seed).permutation(len(tgt))]


@pytest.mark.parametrize("k", [8, 20])
def test_points_exactly_at_matcher_and_outlier_distances(k):
    rng = np.random.default_rng(k)
    tgt = _shuffled(lattice(k), k)
    # 0.5 m from one lattice point (and the next one: also a 2-way tie), 0.5*sqrt(2) m from four, 0.25 m from one
    src = knife_source(k, [(0.5, 0.0), (0.0, 0.5), (0.5, 0.5), (0.25, 0.0)], rng)
    assert np.cumsum(tgt[:, 0], dtype=F32)[-1] == 0 and np.cumsum(tgt[:, 1], dtype=F32)[-1] == 0
    # matcher at 0.5: points at d2 = 0.25 exactly are accepted (<=), those at 0.5 are not
    det = _check(src, tgt, np.eye(3), matcher_max_dist=0.5, outlier_max_dist=-1.0, trim_ratio=-1.0)
    assert (det["d2"] == F32(0.25)).sum() >= 200 and (det["match"] < 0).sum() >= 100
    # MaxDist filter at 0.5: squared compare keeps d2 <= 0.25; raw compare keeps d2 <= 0.5 (the 4-way points too)
    det_sq = _check(src, tgt, np.eye(3), matcher_max_dist=10.0, outlier_max_dist=0.5, trim_ratio=-1.0)
    det_raw = _check(src, tgt, np.eye(3), matcher_max_dist=10.0, outlier_max_dist=0.5, trim_ratio=-1.0, flags=1)
    at_sq = (det_sq["d2"] == F32(0.25)).sum()
    at_raw = (det_raw["d2"] == F32(0.5)).sum()
    assert at_sq >= 200 and at_raw >= 100
    assert det_raw["keep"].sum() == det_sq["keep"].sum() + at_raw


@pytest.mark.parametrize("ratio", [0.5, 0.95, 0.0, 1.0])
def test_many_equal_distances_at_the_trim_quantile(ratio):
    k = 12
    rng = np.random.default_rng(3)
    tgt = _shuffled(lattice(k), 5)
    src = knife_source(k, [(0.25, 0.0)] * 3 + [(0.0, 0.125), (0.5, 0.5)], rng, n_each=80)
    det = _check(src, tgt, np.eye(3), trim_ratio=ratio, outlier_max_dist=-1.0)
    # the quantile element is one of many equal distances: all of them are kept, none beyond
    assert (det["d2"] == det["limit"]).sum() >= 80
    assert det["keep"].sum() == (det["d2"] <= det["limit"]).sum()


def test_ties_between_two_and_four_targets_take_the_lowest_index():
    k = 10
    rng = np.random.default_rng(4)
    tgt = _shuffled(lattice(k), 6)
    src = knife_source(k, [(0.5, 0.0), (0.5, 0.5)], rng, n_each=150)
    det = _check(src, tgt, np.eye(3), trim_ratio=-1.0, outlier_max_dist=-1.0)
    ref = tgt.astype(np.float64)
    d = ((src[:, None, :].astype(np.float64) - ref[None]) ** 2).sum(-1)
    n_min = (d == d.min(1, keepdims=True)).sum(1)
    assert (n_min == 2).sum() >= 100 and (n_min == 4).sum() >= 100
    # the lowest index among the tied targets is not the first one met in a row-major scan of the lattice
    first_in_scan = [min(np.flatnonzero(d[i] == d[i].min()), key=lambda j: (tgt[j, 1], tgt[j, 0])) for i in range(len(src))]
    assert (det["match"] != np.array(first_in_scan)).sum() >= 100
    assert np.array_equal(det["match"], np.argmin(d, 1))


# ------------------------------------------------------------------ random pairs, every setting of the grid
def _pairs():
    out = []
    for seed, ns, nt in ((1, 300, 1200), (2, 500, 2500)):
        s, t, T = synth.make_icp_pair(400 + seed, n_source=ns, n_target=nt)
        g = (T @ synth.se2(0.05 * seed, -0.04, 0.01)).astype(F32)
        out.append((s, t, g))
    return out


@pytest.mark.parametrize("matcher", MATCHER)
@pytest.mark.parametrize("outlier", OUTLIER, ids=[o[0] for o in OUTLIER])
@pytest.mark.parametrize("trim", TRIM)
def test_random_pairs_every_setting(matcher, outlier, trim):
    for s, t, g in _pairs():
        _check(s, t, g, matcher_max_dist=matcher, outlier_max_dist=outlier[1], flags=outlier[2], trim_ratio=trim)


def test_raw_and_squared_outlier_compares_keep_different_sets():
    s, t, g = _pairs()[0]
    g = (g @ synth.se2(1.0, 0.0, 0.0)).astype(F32)  # 1 m off: many distances between 2 and 4 m^2
    sq = _check(s, t, g, outlier_max_dist=2.0, trim_ratio=-1.0)
    raw = _check(s, t, g, outlier_max_dist=2.0, trim_ratio=-1.0, flags=1)
    assert raw["keep"].sum() < sq["keep"].sum()


def test_infinite_matcher_distance_matches_every_point():
    s, t, g = _pairs()[1]
    far = np.c_[np.full(20, 500.0), np.linspace(-300, 300, 20)].astype(F32)
    src = np.concatenate([s, far])
    for md in (float("inf"), 1e9):
        det = _check(src, t, g, matcher_max_dist=md, outlier_max_dist=-1.0, trim_ratio=-1.0)
        assert (det["match"] >= 0).all()
    det = _check(src, t, g)  # shipped 10 m: the far points are unmatched
    assert (det["match"][-20:] < 0).all()


# ------------------------------------------------------------------ settings the matcher cannot honour
def test_yaml_parser_rejects_trim_ratio_above_one_and_nan():
    from sonar_slam_b200.bruce_slam import pcl
    ok = pcl.parse_icp_yaml("outlierFilters:\n  - TrimmedDistOutlierFilter:\n      ratio: 1.0\n")
    assert ok.trim_ratio == 1.0
    for bad in ("outlierFilters:\n  - TrimmedDistOutlierFilter:\n      ratio: 1.5\n",
                "outlierFilters:\n  - TrimmedDistOutlierFilter:\n      ratio: .nan\n",
                "outlierFilters:\n  - MaxDistOutlierFilter:\n      maxDist: .nan\n",
                "matcher:\n  KDTreeMatcher:\n    maxDist: .nan\n",
                "transformationCheckers:\n  - DifferentialTransformationChecker:\n      minDiffRotErr: .nan\n"):
        with pytest.raises(ValueError):
            pcl.parse_icp_yaml(bad)
    # a missing matcher maxDist is libpointmatcher's default, infinity
    assert pcl.parse_icp_yaml("matcher:\n  KDTreeMatcher:\n    knn: 1\n").matcher_max_dist == float("inf")
