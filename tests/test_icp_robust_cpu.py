"""CPU: the RobustOutlierFilter -- the icp.yaml parser, oracle/robust_ref.c's weights against a literal float32
statement and against numpy float64, one weighted iteration against numpy, and the unweighted identity (Huber with k^2
above every kept squared distance equals the chain without it, bit for bit, in both minimisers)."""
import math

import numpy as np
import pytest

from oracle import oracle as orc
from oracle import robust_ref as rr
from oracle import voxel_filter_ref as vfr
from sonar_slam_b200 import _lib, synth
from sonar_slam_b200.bruce_slam import pcl

F32 = np.float32
BASE = ("matcher:\n  KDTreeMatcher:\n    maxDist: 10.0\n"
        "outlierFilters:\n  - MaxDistOutlierFilter:\n      maxDist: 3.0\n{robust}")


def _parse(**p):
    lines = "".join(f"      {k}: {v}\n" for k, v in p.items())
    text = BASE.format(robust="  - RobustOutlierFilter:\n" + (lines or "      {}\n"))
    return pcl.parse_icp_yaml(text)


# ------------------------------------------------------------------ parser
@pytest.mark.parametrize("fct", list(_lib.ROBUST_FCT))
@pytest.mark.parametrize("scale", ["none", "fixed"])
def test_parser_accepts(fct, scale):
    prm = _parse(robustFct=fct, tuning=0.5, scaleEstimator=scale, nbIterationForScale=7)
    r = prm.robust
    assert (r.fct, r.tuning, r.approximation) == (_lib.ROBUST_FCT[fct], F32(0.5), math.inf)
    assert prm.filters is None and prm.outlier_max_dist == F32(3.0)


def test_parser_defaults_and_options():
    r = _parse(scaleEstimator="none").robust
    assert (r.fct, r.tuning, r.approximation) == (_lib.ROBUST_FCT["cauchy"], 1.0, math.inf)
    r = _parse(scaleEstimator="fixed", approximation=4.0, distanceType="point2point", robustFct="tukey").robust
    assert (r.fct, r.approximation) == (_lib.ROBUST_FCT["tukey"], 4.0)
    r = _parse(scaleEstimator="none", approximation=".inf").robust
    assert r.approximation == math.inf
    assert pcl.parse_icp_yaml(BASE.format(robust="")).robust is None


@pytest.mark.parametrize("p", [dict(), dict(scaleEstimator="mad"), dict(scaleEstimator="berg"),
                               dict(scaleEstimator="none", robustFct="student"),
                               dict(scaleEstimator="none", distanceType="point2plane")])
def test_parser_refuses_unimplemented(p):
    with pytest.raises(NotImplementedError):
        _parse(**p)


def test_parser_refuses_a_second_robust_filter():
    one = "  - RobustOutlierFilter:\n      scaleEstimator: none\n"
    with pytest.raises(NotImplementedError, match="second"):
        pcl.parse_icp_yaml(BASE.format(robust=one + one))


@pytest.mark.parametrize("p", [dict(tuning=0), dict(tuning=-1), dict(tuning=".inf"), dict(tuning=".nan"),
                               dict(approximation=".nan"), dict(robustFct="bogus"), dict(scaleEstimator="other"),
                               dict(distanceType="point2line")])
def test_parser_refuses_bad_values(p):
    p = dict(dict(scaleEstimator="none"), **p)
    with pytest.raises(ValueError):
        _parse(**p)


def test_3d_clouds_are_refused_before_any_device_call():
    icp = pcl.ICP()
    icp.params = _parse(scaleEstimator="none")
    with pytest.raises(NotImplementedError, match="RobustOutlierFilter"):
        icp._dim([np.zeros((4, 3), F32)], [np.zeros((4, 3), F32)])
    assert icp._dim([np.zeros((4, 2), F32)], [np.zeros((4, 2), F32)]) == 2


# ------------------------------------------------------------------ weights
def _f(x):
    return F32(x)


def _statement(fct, k, e2):
    """Literal float32 restatement of the weight table (numpy float32 scalars round every operation)."""
    k, e2 = _f(k), _f(e2)
    k2 = k * k
    with np.errstate(all="ignore"):
        if fct == "cauchy":
            return _f(1) / (_f(1) + e2 / k2)
        if fct == "welsch":
            return _f(math.exp(-float(e2 / k2)))
        if fct == "sc":
            return (_f(4) * k2) / ((k + e2) * (k + e2)) if e2 >= k else _f(1)
        if fct == "gm":
            return k2 / ((k + e2) * (k + e2))
        if fct == "tukey":
            return _f(0) if e2 >= k2 else (_f(1) - e2 / k2) * (_f(1) - e2 / k2)
        if fct == "huber":
            return k / np.sqrt(e2) if e2 >= k2 else _f(1)
        return _f(1) / np.sqrt(e2)


def _float64(fct, k, e2):
    k, e2 = float(k), np.float64(e2)
    with np.errstate(all="ignore"):
        return {"cauchy": 1 / (1 + e2 / k ** 2), "welsch": np.exp(-e2 / k ** 2),
                "sc": 4 * k ** 2 / (k + e2) ** 2 if e2 >= k else 1.0, "gm": k ** 2 / (k + e2) ** 2,
                "tukey": 0.0 if e2 >= k ** 2 else (1 - e2 / k ** 2) ** 2,
                "huber": k / np.sqrt(e2) if e2 >= k ** 2 else 1.0, "L1": 1 / np.sqrt(e2)}[fct]


E2 = np.concatenate([[0.0, 1e-30, 1e-8, 0.01, 0.0025, 0.04, 0.05, 0.25, 0.3, 1.0, 9.0, 1e30, np.inf],
                     np.random.default_rng(0).uniform(0, 2, 200) ** 3]).astype(F32)


@pytest.mark.parametrize("k", [0.05, 0.3, 1.0, 2.5])
@pytest.mark.parametrize("fct", list(rr.FCT))
def test_weights_against_statement_and_float64(fct, k):
    w = rr.weights(E2, rr.Robust(fct, k))
    want = np.array([_statement(fct, k, e) for e in E2], F32)
    assert np.array_equal(w.view(np.uint32), want.view(np.uint32)), fct
    ref = np.array([_float64(fct, F32(k), e) for e in E2])
    fin = np.isfinite(ref) & (ref > 1e-30)
    # float32 rounding, amplified by welsch's exponent and by tukey's 1 - e2 / k2 near k2
    tol = 1e-6 + 1e-6 * (1 + np.abs(np.log(ref[fin]))) * ref[fin]
    assert np.all(np.abs(w[fin] - ref[fin]) <= tol)
    assert np.array_equal(np.isinf(w), np.isinf(ref))


@pytest.mark.parametrize("fct", list(rr.FCT))
def test_approximation_cut_off(fct):
    w = rr.weights(E2, rr.Robust(fct, 0.5, 0.3))
    assert np.all(w[E2 >= F32(0.3)] == 0)
    assert np.array_equal(w[E2 < F32(0.3)], rr.weights(E2[E2 < F32(0.3)], rr.Robust(fct, 0.5)))


# ------------------------------------------------------------------ iterations
def test_one_weighted_iteration_against_numpy():
    """One iteration, no other filter (MaxDist and Trimmed off): the weighted point-to-point fit of the matches, in
    float64 -- close to the oracle's float32 sequential sums."""
    src, tgt, T = synth.make_icp_pair(5, n_source=300, n_target=900)
    g = T.astype(F32)
    prm = orc.IcpParams(outlier_max_dist=-1.0, trim_ratio=-1.0, max_iterations=1, smooth_length=0)
    rob = rr.Robust("cauchy", 0.1)
    got = rr.icp(src, tgt, g, prm, robust=rob)
    assert got["status"] == 0 and got["iterations"] == 1
    mean = tgt.astype(np.float64).mean(0)
    ref = tgt.astype(np.float64) - mean
    rd = (src.astype(np.float64) @ g[:2, :2].T.astype(np.float64)) + g[:2, 2] - mean
    d2 = ((rd[:, None, :] - ref[None, :, :]) ** 2).sum(-1)
    j = d2.argmin(1)
    e2 = d2[np.arange(len(rd)), j]
    keep = e2 <= 100.0
    w = 1 / (1 + e2 / 0.01) * keep
    W = w.sum()
    mp, mq = (w[:, None] * rd).sum(0) / W, (w[:, None] * ref[j]).sum(0) / W
    M = ((w[:, None] * (ref[j] - mq)).T @ (rd - mp))
    ang = math.atan2(M[1, 0] - M[0, 1], M[0, 0] + M[1, 1])
    R = np.array([[math.cos(ang), -math.sin(ang)], [math.sin(ang), math.cos(ang)]])
    t = mq - R @ mp
    Tit = np.eye(3)
    Tit[:2, :2], Tit[:2, 2] = R, t
    Tm = np.eye(3)
    Tm[:2, 2] = mean
    want = Tm @ Tit @ np.linalg.inv(Tm) @ g.astype(np.float64)
    assert got["inliers"] == int((w != 0).sum())
    assert np.abs(got["T"] - want).max() < 2e-4


@pytest.mark.parametrize("checkers", [{}, dict(max_iterations=20, smooth_length=0)])
@pytest.mark.parametrize("minimizer", [0, 1])
def test_huber_identity_equals_the_chain_without_it(minimizer, checkers):
    """Huber with k^2 > maxDist^2: every kept pair weighs exactly 1, so the weighted chain is the unweighted one."""
    prm = orc.IcpParams(minimizer=minimizer, **checkers)
    flt = vfr.IcpFilters(min_dist=0.01, reading=[(vfr.MAX_DIST, -1, 20.0)])
    for seed in range(3):
        s, t, T = synth.make_icp_pair(70 + seed, n_source=400, n_target=1200)
        g = T.astype(F32)
        for f in (None, flt):
            a = rr.icp(s, t, g, prm, f, rr.Robust("huber", 3.5))
            b = vfr.icp(s, t, g, prm, f)
            assert (a["status"], a["iterations"], a["inliers"]) == (b["status"], b["iterations"], b["inliers"])
            assert np.array_equal(a["T"].view(np.uint32), b["T"].view(np.uint32))
            assert b["status"] == 0 or f is not None


def test_ctypes_struct_matches_the_oracle_block():
    assert _lib.IcpRobust._fields_ == [(n, t) for n, t in rr.Robust._fields_]
    assert _lib.ROBUST_FCT == rr.FCT
