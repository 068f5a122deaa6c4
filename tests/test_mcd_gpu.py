"""GPU: the batched MinCovDet kernel (csrc/mcd.cu) against scikit-learn's MinCovDet(support_fraction=0.8) itself, and
SLAM.compute_icp_with_cov_batch against the sequential compute_icp_with_cov calls.  The device gets the trial supports
that a RandomState with the same seed hands sklearn (sonar_slam_b200/mcd.py: draw_trial_supports)."""
import os
import types

import numpy as np
import pytest

from sonar_slam_b200 import _lib, mcd

pytestmark = pytest.mark.gpu
sk = pytest.importorskip("sklearn.covariance")

RTOL, ATOL = 1e-9, 1e-15
MSG = {mcd.OK: "success", mcd.ZERO_COV: "Failed to calculate covariance",
       mcd.TOO_FEW: "Too few samples for covariance computation"}


class _Replay(np.random.RandomState):
    def __init__(self, supports, n):
        super().__init__(0)
        self.rows = [np.concatenate([s, np.setdiff1d(np.arange(n), s)]) for s in supports]

    def permutation(self, x):
        return self.rows.pop(0)


def _sklearn(X, rs):
    try:
        f = sk.MinCovDet(store_precision=False, support_fraction=0.8, random_state=rs).fit(X)
    except ValueError:
        return dict(status=mcd.ZERO_COV)
    return dict(status=mcd.OK, location=np.asarray(f.location_, np.float64), covariance=f.covariance_,
                raw=f.raw_support_, support=f.support_, raw_covariance=f.raw_covariance_)


def _permuted(X, sup, q, seed):
    """sklearn on a row permutation of X, the trial supports permuted to match; supports mapped back to X's rows"""
    n, h = len(X), mcd.support_size(len(X))
    perm = np.arange(n) if q == 0 else np.random.default_rng(seed).permutation(n)
    inv = np.argsort(perm)
    w = _sklearn(X[perm], _Replay([inv[sup[t, :h]] for t in range(mcd.TRIALS)], n))
    if w["status"] == mcd.OK:
        w["raw"], w["support"] = w["raw"][inv], w["support"][inv]
    return w


def _device(sets, supports, float32):
    X, n = mcd.pack(sets)
    return mcd.mincovdet_host(X, n, np.stack(supports), float32=float32)


def _rows(X, mask):
    """the selected rows as a sorted multiset (swapping two bit-identical samples is no difference)"""
    r = np.asarray(X, np.float64)[mask]
    return r[np.lexsort(r.T[::-1])]


def _generic_set(rng, float32):
    n = int(rng.integers(5, 33))
    sxy = 10 ** rng.uniform(-3, np.log10(0.5))
    sth = 10 ** rng.uniform(-4, np.log10(0.05))
    X = rng.normal([rng.normal(0, 3), rng.normal(0, 3), rng.uniform(-1, 1)], [sxy, sxy, sth], (n, 3))
    k = int(round(rng.uniform(0, 0.4) * n))
    if k:
        X[:k] += rng.normal(0, 1, (k, 3)) * [sxy, sxy, sth] * rng.uniform(5, 50)
    X = X[rng.permutation(n)]
    return X.astype(np.float32) if float32 else X


@pytest.mark.parametrize("float32,count", [(False, 2000), (True, 500)])
def test_generic_sets_equal_sklearn(gpu_ctx, float32, count):
    rng = np.random.default_rng(2024 + float32)
    sets = [_generic_set(rng, float32) for _ in range(count)]
    sup = [mcd.draw_trial_supports(len(X), np.random.RandomState(s)) for s, X in enumerate(sets)]
    got = _device(sets, sup, float32)
    bad, tied = [], 0
    for s, X in enumerate(sets):
        g = {k: v[s] for k, v in got.items()}
        why = _differs(X, g, _sklearn(X, np.random.RandomState(s)))
        if why and len(X) <= 6 and why[0] != "status":
            # h = int(0.8 n) = 4 = p + 1 for n = 5, 6: under the covariance of h rows, each of those rows has Mahalanobis
            # distance exactly h - 1 = 3, so a C-step that keeps only some of them chooses among exact ties, and the
            # choice is made by rounding (LAPACK's eigh and numpy's argpartition on the host, Jacobi and the rank here).
            # Such a set may end in a different support than sklearn's; the status must still agree, and such sets
            # must stay rare.
            tied, why = tied + 1, None
        if why:
            bad.append((s, len(X)) + why)
    assert not bad, bad[:10]
    assert tied <= count // 100, tied
    assert (got["status"] == mcd.OK).sum() > 0.95 * count


def _differs(X, g, w):
    """None when the device result g equals sklearn's w: status, raw and final supports as multisets of rows,
    location and covariance within RTOL / ATOL"""
    if g["status"] != w["status"]:
        return ("status", int(g["status"]), w["status"])
    if w["status"] != mcd.OK:
        return None
    n = len(X)
    if not np.array_equal(_rows(X, mcd.mask_rows(g["raw_support"], n)), _rows(X, w["raw"])):
        return ("raw support",)
    if not np.array_equal(_rows(X, mcd.mask_rows(g["support"], n)), _rows(X, w["support"])):
        return ("support",)
    if not (np.allclose(g["location"], w["location"], rtol=RTOL, atol=ATOL)
            and np.allclose(g["covariance"], w["covariance"], rtol=RTOL, atol=ATOL)):
        return ("values", np.abs(g["location"] - w["location"]).max(), np.abs(g["covariance"] - w["covariance"]).max())
    return None


def _finish(status, loc, cov):
    """compute_icp_with_cov's message, whether it substitutes the default covariance, and the location"""
    if status != mcd.OK:
        return MSG[status], None, None
    from sonar_slam_b200.bruce_slam.slam import Pose2
    m = Pose2(*loc)
    cov = np.array(cov)
    R = m.matrix()[:2, :2]
    cov[:2, :] = R.T.dot(cov[:2, :])
    cov[:, :2] = cov[:, :2].dot(R)
    return "success", bool(np.linalg.det(cov) < np.linalg.det(np.diag([0.1, 0.1, 0.01]) ** 2)), np.asarray(loc)


def _same(a, b, location=True):
    return a[0] == b[0] and a[1] == b[1] and (not location or a[2] is None or np.allclose(a[2], b[2], rtol=0, atol=1e-9))


def _degenerate_sets(rng):
    out = []
    for _ in range(6):
        n = int(rng.integers(6, 33))
        h = mcd.support_size(n)
        base = rng.normal([1.0, -0.5, 0.2], [0.05, 0.05, 0.005], (n, 3))
        for k in sorted({max(1, h - 2), h, n}):          # k identical rows: k < h, k = h, k = n
            X = base.copy()
            X[:k] = base[0]
            out.append(X[rng.permutation(n)])
        X = base.copy()
        X[:, 2] = base[0, 2]                               # constant theta column
        out.append(X)
        out.append(base[rng.integers(0, 3, n)])            # three distinct rows repeated
        X = rng.normal([1.0, -0.5, 0.2], [1e-4, 1e-4, 1e-5], (n, 3)) * [rng.uniform(0.7, 1.4), 1, 1]
        out.append(X)                                      # raw covariance near allclose's 1e-8
    return [X.astype(np.float32) for X in out]


def test_degenerate_sets_match_sklearns_decisions(gpu_ctx):
    rng = np.random.default_rng(99)
    sets = _degenerate_sets(rng)
    sup = [mcd.draw_trial_supports(len(X), np.random.RandomState(s)) for s, X in enumerate(sets)]
    got = _device(sets, sup, True)
    bad, agreed, singular = [], 0, 0
    for s, X in enumerate(sets):
        ws = [_permuted(X, sup[s], q, 1000 * s + q) for q in range(4)]   # sklearn on row permutations of the set
        answers = [_finish(w["status"], w.get("location"), w.get("covariance")) for w in ws]
        mine = _finish(int(got["status"][s]), got["location"][s], got["covariance"][s])
        # a raw covariance that is singular up to rounding (eigenvalues ~1e-20 next to 1e-4) came out of a choice
        # among supports whose log-dets are rounding noise (-inf or a finite value, by the sign of that noise): which of
        # them wins is not reproducible across implementations, so there only the message and the default-covariance
        # decision are compared
        ev = [np.linalg.eigvalsh(w["raw_covariance"]) for w in ws if w["status"] == mcd.OK]
        loc = not any(e[0] <= 1e-12 * e[-1] for e in ev)
        singular += not loc
        if all(_same(a, answers[0], loc) for a in answers):
            agreed += 1
            if not _same(mine, answers[0], loc):
                bad.append((s, mine[:2], answers[0][:2]))
        elif not any(_same(mine, a, loc) for a in answers):
            bad.append((s, "matches none", mine[:2], [a[:2] for a in answers]))
    assert not bad, bad
    assert agreed >= len(sets) // 2 and singular < len(sets)


def _stub_icp(T, ok):
    msgs = ["success" if o else "ErrorMnimizer: no point to minimize" for o in ok]
    return types.SimpleNamespace(compute_pairs=lambda s, t, g: [dict(messages=msgs[:len(x)], T=T[:len(x)]) for x in g])


def test_golden_fixture_through_the_device(gpu_ctx, golden_dir):
    from sonar_slam_b200.bruce_slam import slam
    g = np.load(os.path.join(golden_dir, "slam_host.npz"))
    s = slam.SLAM()
    s.icp = _stub_icp(g["cov_T"], g["cov_ok"])
    np.random.seed(1234)   # the seed the fixture's MinCovDet fit drew under (tools/make_golden.py)
    msg, m, cov, samples = s.compute_icp_with_cov_batch([(g["kf0_points"], g["kf1_points"],
                                                         [slam.Pose2(0.01 * i, 0, 0) for i in range(14)])])[0]
    assert msg == "success" and np.array_equal(samples, g["cov_samples"])
    assert np.allclose([m.x(), m.y(), m.theta()], g["cov_mean"], rtol=RTOL, atol=ATOL)
    assert np.allclose(cov, g["cov_cov"], rtol=RTOL, atol=ATOL)


def test_end_to_end_against_sequential_sklearn_path(gpu_ctx, icp_yaml):
    from sonar_slam_b200 import synth
    from sonar_slam_b200.bruce_slam.slam import SLAM, Pose2
    s = SLAM()
    s.icp.loadFromYaml(icp_yaml)
    rng = np.random.default_rng(5)
    problems = []
    for c in range(50):
        src, tgt, T = synth.make_icp_pair(300 + c, n_source=1500, n_target=4000)
        th = np.arctan2(T[1, 0], T[0, 0])
        problems.append((src, tgt, [Pose2(*(np.array([T[0, 2], T[1, 2], th]) + rng.normal(0, [0.2, 0.2, 0.02])))
                                    for _ in range(30)]))
    np.random.seed(77)
    want = [s.compute_icp_with_cov(*p) for p in problems]
    np.random.seed(77)
    got = s.compute_icp_with_cov_batch(problems)
    assert sum(w[0] == "success" for w in want) >= 40
    for w, o in zip(want, got):
        assert o[0] == w[0]
        if w[0] != "success":
            continue
        assert o[3].dtype == w[3].dtype and np.array_equal(o[3], w[3])
        assert np.allclose([o[1].x(), o[1].y(), o[1].theta()], [w[1].x(), w[1].y(), w[1].theta()], rtol=RTOL, atol=ATOL)
        assert np.allclose(o[2], w[2], rtol=RTOL, atol=ATOL)


def test_one_batch_equals_one_problem_per_call(gpu_ctx):
    import torch
    from sonar_slam_b200 import ops
    rng = np.random.default_rng(3)
    sets = [_generic_set(rng, False) for _ in range(4096)]
    sets[7] = sets[7][:3]                                            # too few
    sets[11] = np.repeat(sets[11][:1], len(sets[11]), 0)             # zero covariance
    sup = [mcd.draw_trial_supports(max(len(X), 5), np.random.RandomState(s)) for s, X in enumerate(sets)]
    X, n = mcd.pack(sets)
    S = np.stack(sup)
    dev = ops.mincovdet(torch.from_numpy(X).cuda(), torch.from_numpy(n).cuda(), torch.from_numpy(S).cuda())
    torch.cuda.synchronize()
    one = [mcd.mincovdet_host(X[p:p + 1], n[p:p + 1], S[p:p + 1]) for p in range(len(sets))]
    for key in ("location", "covariance", "raw_support", "support", "status"):
        a = dev[key].cpu().numpy()
        b = np.concatenate([o[key] for o in one])
        assert np.array_equal(a.view(np.uint8), b.astype(a.dtype).view(np.uint8)), key
    st = dev["status"].cpu().numpy()
    assert st[7] == mcd.TOO_FEW and st[11] == mcd.ZERO_COV


def test_argument_errors(gpu_ctx):
    X, n = mcd.pack([np.zeros((5, 3))])
    with pytest.raises(_lib.SonarFEError):
        mcd.mincovdet_host(X, np.array([33], np.int32), mcd.draw_trial_supports(5)[None])
    bad = mcd.draw_trial_supports(5)[None].copy()
    bad[0, 3, 1] = bad[0, 3, 0]                                      # a repeated row
    r = mcd.mincovdet_host(np.random.default_rng(0).normal(size=X.shape), n, bad)
    assert r["status"][0] == mcd.BAD_SUBSET
