"""CPU-only tests of the host side of the device MinCovDet (sonar_slam_b200/mcd.py) and of
SLAM.compute_icp_with_cov_batch: the trial supports and constants handed to the kernel are sklearn's own, and the batch
method returns what the sequential compute_icp_with_cov calls return.  ICP answers and the MinCovDet entry point are
served by stand-ins here (the MCD stand-in is sklearn itself, replaying the supports it is passed), so what is tested is
the Python around the two device calls."""
import os
import types

import numpy as np
import pytest

sklearn_cov = pytest.importorskip("sklearn.covariance")
from sklearn.covariance._robust_covariance import _consistency_factor  # noqa: E402

from sonar_slam_b200 import mcd  # noqa: E402
from sonar_slam_b200.bruce_slam import slam  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden", "slam_host.npz")


class _Recording(np.random.RandomState):
    """RandomState that records every permutation() call sklearn makes."""

    def __init__(self, seed):
        super().__init__(seed)
        self.calls = []

    def permutation(self, x):
        p = super().permutation(x)
        self.calls.append((x, p.copy()))
        return p


class _Replay(np.random.RandomState):
    """RandomState whose permutation() calls return the given trial supports, in order."""

    def __init__(self, supports, n):
        super().__init__(0)
        self.rows = [np.concatenate([s, np.setdiff1d(np.arange(n), s)]) for s in supports]

    def permutation(self, x):
        return self.rows.pop(0)


def sklearn_mincovdet_host(samples, n, subsets, float32=False, ctx=None):
    """Stand-in for mcd.mincovdet_host with its contract: sklearn MinCovDet on every problem, started from the passed
    supports."""
    P = len(n)
    loc, cov = np.full((P, 3), np.nan), np.full((P, 3, 3), np.nan)
    raw, sup, st = np.zeros(P, np.uint32), np.zeros(P, np.uint32), np.zeros(P, np.int32)
    for p in range(P):
        k = int(n[p])
        h = mcd.support_size(k)
        X = samples[p, :k].astype(np.float32 if float32 else np.float64)
        rs = _Replay([subsets[p, t, :h].astype(np.int64) for t in range(mcd.TRIALS)], k)
        try:
            f = sklearn_cov.MinCovDet(store_precision=False, support_fraction=0.8, random_state=rs).fit(X)
        except ValueError:
            st[p] = mcd.ZERO_COV
            continue
        assert not rs.rows
        loc[p], cov[p] = f.location_, f.covariance_
        raw[p] = int(np.sum(f.raw_support_ << np.arange(k)))
        sup[p] = int(np.sum(f.support_ << np.arange(k)))
    return dict(location=loc, covariance=cov, raw_support=raw, support=sup, status=st)


@pytest.mark.parametrize("n", range(5, 33))
def test_trial_supports_are_sklearns_draws(n):
    rng = np.random.default_rng(n)
    X = rng.normal(0, [0.1, 0.1, 0.01], (n, 3))
    rec = _Recording(100 + n)
    sklearn_cov.MinCovDet(store_precision=False, support_fraction=0.8, random_state=rec).fit(X)
    assert len(rec.calls) == mcd.TRIALS and all(x == n for x, _ in rec.calls)
    h = mcd.support_size(n)
    assert h == int(0.8 * n)
    got = mcd.draw_trial_supports(n, np.random.RandomState(100 + n))
    assert got.shape == (mcd.TRIALS, mcd.MAX_SAMPLES) and got.dtype == np.int8
    for t, (_, p) in enumerate(rec.calls):
        assert np.array_equal(got[t, :h], p[:h]) and (got[t, h:] == -1).all()
    # random_state=None: the same draws from numpy's global generator
    np.random.seed(100 + n)
    assert np.array_equal(mcd.draw_trial_supports(n), got)


def test_constants_are_the_installed_librarys():
    from scipy.stats import chi2
    c, c_rw, cut = mcd.constants()
    assert c.shape == (33,)
    for n in range(5, 33):
        assert c[n] == _consistency_factor(3, int(0.8 * n) / n)
    assert c_rw == _consistency_factor(3, 0.975) and cut == chi2(3).isf(0.025)


def _candidates():
    """(source, target, guesses, icp messages, icp T) per candidate: the golden one, then synthetic ones that reach
    every branch of compute_icp_with_cov."""
    g = np.load(GOLD)
    ok_msgs = ["success" if ok else "ErrorMnimizer: no point to minimize" for ok in g["cov_ok"]]
    rng = np.random.default_rng(7)
    out = []

    def add(T, msgs=None):
        src = rng.normal(0, 5, (50 + len(out), 2)).astype(np.float32)   # distinct clouds identify the candidate
        tgt = rng.normal(0, 5, (80, 2)).astype(np.float32)
        guesses = [slam.Pose2(0.01 * i, 0.0, 0.0) for i in range(len(T))]
        out.append((src, tgt, guesses, msgs or ["success"] * len(T), np.asarray(T, np.float32)))

    def Ts(poses):
        return [slam.Pose2(*p).matrix() for p in poses]

    out.append((g["kf0_points"], g["kf1_points"], [slam.Pose2(0.01 * i, 0.0, 0.0) for i in range(14)], ok_msgs,
                g["cov_T"]))
    out.append((g["kf0_points"][:40], g["kf1_points"], [slam.Pose2(0.01 * i, 0.0, 0.0) for i in range(5)],
                ok_msgs[:5], g["cov_T"][:5]))                                          # 4 successes: too few
    for k in range(6):                                                                # generic, with outliers
        nk = int(rng.integers(5, 31))
        poses = rng.normal([1.0, -0.5, 0.1], [0.05, 0.05, 0.01], (nk, 3))
        poses[: nk // 5] += rng.normal(0, [0.5, 0.5, 0.1], (nk // 5, 3))
        msgs = ["success" if rng.random() > 0.1 else "no outlier to filter" for _ in range(nk)]
        add(Ts(poses), msgs)
    add(Ts([[0.3, 0.2, 0.05]] * 30))                                                 # all identical: ValueError
    add(Ts([[0.3, 0.2, 0.05]] * 26 + list(rng.normal([0.3, 0.2, 0.05], 0.1, (4, 3)))))  # > h identical: ValueError
    add(Ts(rng.normal([2.0, 1.0, 0.3], [3e-3, 3e-3, 3e-4], (20, 3))))                # tight: default covariance
    add(Ts(rng.normal([2.0, 1.0, 0.3], [1e-4, 1e-4, 1e-5], (3, 3))))                 # 3 samples: too few
    return out


def _serve(s, cands):
    by_src = {np.asarray(c[0], np.float32).tobytes(): c for c in cands}

    def compute_batch(src, tgt, guesses):
        c = by_src[np.asarray(src, np.float32).tobytes()]
        assert len(guesses) == len(c[2])
        return dict(messages=list(c[3]), T=c[4])

    def compute_pairs(sources, targets, guesses):
        assert len(sources) == len(targets) == len(guesses) == len(cands)
        return [compute_batch(a, b, g) for a, b, g in zip(sources, targets, guesses)]

    s.icp = types.SimpleNamespace(compute_batch=compute_batch, compute_pairs=compute_pairs)


def _host_slam():
    s = slam.SLAM.__new__(slam.SLAM)   # no ICP objects: nothing here may touch the device
    s.point_resolution, s.point_noise = 0.5, 0.5
    s.icp_odom_sigmas = np.array([0.1, 0.1, 0.01])
    return s


def test_batch_equals_sequential_reference_calls(monkeypatch):
    monkeypatch.setattr(mcd, "mincovdet_host", sklearn_mincovdet_host)
    cands = _candidates()
    s = _host_slam()
    _serve(s, cands)
    np.random.seed(1234)
    want = [s.compute_icp_with_cov(src, tgt, gs) for src, tgt, gs, _, _ in cands]
    np.random.seed(1234)
    got = s.compute_icp_with_cov_batch([(src, tgt, gs) for src, tgt, gs, _, _ in cands])
    after = np.random.random()
    np.random.seed(1234)
    [s.compute_icp_with_cov(src, tgt, gs) for src, tgt, gs, _, _ in cands]
    assert after == np.random.random()            # the batch drew exactly what the sequence draws
    msgs = [w[0] for w in want]
    assert msgs.count("success") >= 6 and msgs.count("Failed to calculate covariance") == 2
    assert msgs.count("Too few samples for covariance computation") == 2
    assert any(w[0] == "success" and np.array_equal(w[2], np.diag(s.icp_odom_sigmas) ** 2) for w in want)
    assert len(got) == len(want)
    for w, o in zip(want, got):
        assert o[0] == w[0]
        if w[0] != "success":
            assert o[1:] == (None, None, None)
            continue
        assert [o[1].x(), o[1].y(), o[1].theta()] == [w[1].x(), w[1].y(), w[1].theta()]
        assert o[2].dtype == w[2].dtype and np.array_equal(o[2], w[2])
        assert o[3].dtype == w[3].dtype and np.array_equal(o[3], w[3])
    # the golden candidate is the reference's own answer (tests/golden/slam_host.npz)
    g = np.load(GOLD)
    assert np.array_equal(got[0][3], g["cov_samples"])
    assert np.allclose([got[0][1].x(), got[0][1].y(), got[0][1].theta()], g["cov_mean"], rtol=0, atol=1e-12)
    assert np.allclose(got[0][2], g["cov_cov"], rtol=1e-12, atol=0)


def test_batch_rejects_more_guesses_than_the_kernel_holds():
    s = _host_slam()
    with pytest.raises(ValueError):
        s.compute_icp_with_cov_batch([(np.zeros((5, 2)), np.zeros((5, 2)), [slam.Pose2()] * 33)])
    assert s.compute_icp_with_cov_batch([]) == []
