"""CPU-only: the 3-D ICP oracle (oracle/icp3_ref.c) -- its SVD, quaternion and nearest-neighbour pieces, its chain
against an independent float64 arm, its statuses, the planar case -- and `pcl.ICP`'s argument checks on [N,3] clouds."""
import numpy as np
import pytest
from scipy.spatial import cKDTree
from scipy.spatial.transform import Rotation

from oracle import cloud3_ref, icp3_ref as o3, oracle as orc
from oracle.oracle import IcpParams
from sonar_slam_b200 import synth
from sonar_slam_b200.bruce_slam import pcl

FIXED20 = dict(max_iterations=20, smooth_length=0)


def _structured():
    rng = np.random.default_rng(7)
    ms = [np.diag([3.0, 2.0, 1.0]), np.diag([1.0, 2.0, 3.0]), np.diag([-1.0, 2.0, -3.0]), np.zeros((3, 3)),
          np.eye(3), -np.eye(3), np.diag([1.0, 1.0, 1.0 + 1e-7]), np.diag([1.0, 0.0, 0.0])]
    for perm in ([0, 2, 1], [1, 0, 2], [2, 0, 1], [1, 2, 0], [2, 1, 0]):
        ms.append(np.eye(3)[perm] * np.array([1.0, 2.0, 3.0]))
    for _ in range(20):
        a, b, c, d = rng.normal(size=(4, 3))
        ms += [np.outer(a, b), np.outer(a, b) + np.outer(c, d)]  # rank 1 and 2
        m = rng.normal(size=(3, 3))
        ms += [-m, m * 1e-30, m * 1e30]
        refl = Rotation.random(random_state=rng).as_matrix() @ np.diag([1.0, 1.0, -1.0])  # det -1: the fix applies
        ms.append(refl * rng.uniform(0.5, 2.0, 3))
    return [np.asarray(m, np.float32) for m in ms]


def _check_svd(M, tol):
    U, S, V, sweeps = o3.svd3(M)
    assert 1 <= sweeps <= 32
    I = np.eye(3)
    assert np.abs(U.astype(np.float64).T @ U - I).max() < 1e-5 and np.abs(V.astype(np.float64).T @ V - I).max() < 1e-5
    scale = max(float(np.abs(M).max()), np.finfo(np.float32).tiny)
    assert np.abs((U.astype(np.float64) * S) @ V.T - M).max() <= tol * scale
    assert (S >= 0).all() and S[0] >= S[1] >= S[2]
    assert np.abs(S - np.linalg.svd(M.astype(np.float64), compute_uv=False)).max() <= tol * scale
    R, fixed = o3.rot3(M)
    assert abs(np.linalg.det(R.astype(np.float64)) - 1.0) < 1e-5
    return U, S, V, R, fixed


def test_svd3_on_random_and_structured_matrices():
    # float32 tolerance: a few dozen rotations of rounded coefficients, relative to the largest |coefficient|
    tol = 2e-6
    rng = np.random.default_rng(0)
    worst = 0.0
    for _ in range(10000):
        M = rng.normal(size=(3, 3)).astype(np.float32) * np.float32(10.0 ** rng.uniform(-3, 3))
        U, S, V, R, fixed = _check_svd(M, tol)
        if S[2] > 0.05 * S[0] and S[1] - S[2] > 0.05 * S[0] and S[0] - S[1] > 0.05 * S[0]:
            # float64 Kabsch with Sorkine's fix
            u, s, vt = np.linalg.svd(M.astype(np.float64))
            if np.linalg.det(u @ vt) < 0:
                vt[2] *= -1
            worst = max(worst, float(np.abs(R - u @ vt).max()))
    assert worst < 1e-4, worst
    print(f"well-conditioned rotations vs float64 Kabsch: max |dR| {worst:.2e}")
    fixes = 0
    for M in _structured():
        U, S, V, R, fixed = _check_svd(M, tol)
        fixes += fixed == 1
    assert fixes >= 20  # the reflection-inducing matrices


def test_svd3_zero_and_non_finite():
    U, S, V, n = o3.svd3(np.zeros((3, 3)))
    assert n == 1 and (S == 0).all() and (U == np.eye(3)).all() and (V == np.eye(3)).all()
    assert (o3.rot3(np.zeros((3, 3)))[0] == np.eye(3)).all()
    for bad in (np.nan, np.inf):
        M = np.eye(3, dtype=np.float32)
        M[1, 2] = bad
        assert o3.svd3(M)[3] == -1
        R, fixed = o3.rot3(M)
        assert fixed == -1 and (R == np.eye(3)).all()


def _rot_to_quat_2d(T):
    """oracle/icp_ref.c rot_to_quat (w, z of a 2-D rotation embedded in 3x3), float32 scalar by scalar"""
    f = np.float32
    m00, m01, m10, m11 = f(T[0, 0]), f(T[0, 1]), f(T[1, 0]), f(T[1, 1])
    t = (m00 + m11) + f(1.0)
    if t > 0:
        t = np.sqrt(t + f(1.0))
        w = f(0.5) * t
        t = f(0.5) / t
        return w, (m10 - m01) * t
    t = np.sqrt(((f(1.0) - m00) - m11) + f(1.0))
    z = f(0.5) * t
    t = f(0.5) / t
    return (m10 - m01) * t, z


def test_quaternion_and_angular_distance():
    rng = np.random.default_rng(1)
    for _ in range(500):
        a, b = Rotation.random(2, random_state=rng)
        qa = o3.quat3(a.as_matrix().astype(np.float32))
        qb = o3.quat3(b.as_matrix().astype(np.float32))
        want = a.as_quat()[[3, 0, 1, 2]]
        assert min(np.abs(qa - want).max(), np.abs(qa + want).max()) < 1e-6
        assert abs(o3.angular_distance3(qa, qb) - (a * b.inv()).magnitude()) < 2e-5
    for th in np.r_[rng.uniform(-np.pi, np.pi, 200), 0.0, np.pi, -np.pi, np.pi / 2]:
        c, s = np.float32(np.cos(th)), np.float32(np.sin(th))
        T = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], np.float32)
        w, z = _rot_to_quat_2d(T)
        q = o3.quat3(T)
        assert q[1] == 0 and q[2] == 0
        assert np.float32(q[0]).tobytes() == np.float32(w).tobytes() and np.float32(q[3]).tobytes() == np.float32(z).tobytes()
        assert o3.det3(T) == np.float32(c * c + s * s) or abs(o3.det3(T) - 1) < 1e-6


def test_nn3_is_exact_with_ties_to_the_lower_index():
    rng = np.random.default_rng(2)
    clouds = [rng.normal(size=(3000, 3)),
              np.c_[rng.normal(size=(2000, 2)) * 0.2, rng.uniform(-20, 20, 2000)],  # a tall column
              np.round(rng.uniform(-2, 2, (2000, 3)) * 4) / 4,                      # coincident points and ties
              np.c_[rng.normal(size=(2000, 2)), np.zeros(2000)]]                    # planar
    for ref in clouds:
        ref = ref.astype(np.float32)
        q = np.r_[ref[:300] + 0.0, rng.normal(size=(700, 3)) * 2, np.round(rng.uniform(-2, 2, (300, 3)) * 8) / 8]
        q = q.astype(np.float32)
        for md in (0.25, 1.0, 50.0):
            ids, d = o3.nn3_match(ref, q, md)
            bi, bd = cloud3_ref.match3(ref, q, md)
            assert np.array_equal(ids, bi[0]) and np.array_equal(d, bd[0])


def _np_icp3(src, tgt, guess, iters=20, max_dist=10.0, out_dist=3.0, ratio=0.8):
    """The same chain in float64: numpy means and SVD, cKDTree neighbours"""
    src, tgt = src.astype(np.float64), tgt.astype(np.float64)
    m = tgt.mean(0)
    ref = tgt - m
    tree = cKDTree(ref)
    T0 = np.eye(4)
    T0[:3, 3] = -m
    T0 = T0 @ guess
    reading = src @ T0[:3, :3].T + T0[:3, 3]
    Ti = np.eye(4)
    for _ in range(iters):
        step = reading @ Ti[:3, :3].T + Ti[:3, 3]
        d, j = tree.query(step, distance_upper_bound=max_dist)
        fin = np.isfinite(d)
        d2 = d ** 2
        lim = np.sort(d2[fin])[int(fin.sum() * ratio)]
        keep = fin & (d2 <= out_dist ** 2) & (d2 <= lim)
        p, r = step[keep], ref[j[keep]]
        mp, mr = p.mean(0), r.mean(0)
        U, _, Vt = np.linalg.svd((r - mr).T @ (p - mp))
        if np.linalg.det(U @ Vt) < 0:
            Vt[2] *= -1
        dT = np.eye(4)
        dT[:3, :3] = U @ Vt
        dT[:3, 3] = mr - dT[:3, :3] @ mp
        Ti = dT @ Ti
    Tm = np.eye(4)
    Tm[:3, 3] = m
    return Tm @ Ti @ T0


def test_oracle_against_float64_arm_and_ground_truth():
    # Bound: the float32 sequential sums move the fit by up to ~2e-3 on these problems (measured 1e-5 .. 2.3e-3 over
    # seeds 0-11); a pair whose trimmed set changes by one point can differ more, hence 1e-2.
    bound = 1e-2
    errs, rot, tr = [], [], []
    for seed in range(8):
        src, tgt, T_gt = synth.make_icp_pair3(seed)
        r = o3.icp3(src, tgt, params=IcpParams(**FIXED20))
        assert r["status"] == 0 and r["iterations"] == 20
        errs.append(float(np.abs(r["T"] - _np_icp3(src, tgt, np.eye(4))).max()))
        r = o3.icp3(src, tgt, params=IcpParams(max_iterations=100, smooth_length=0))
        E = np.linalg.inv(T_gt) @ r["T"]
        rot.append(float(np.arccos(np.clip((np.trace(E[:3, :3]) - 1) / 2, -1, 1))))
        tr.append(float(np.linalg.norm(E[:3, 3])))
    hist, edges = np.histogram(errs, bins=[0, 1e-5, 1e-4, 1e-3, 3e-3, 1e-2, np.inf])
    print("oracle vs float64 arm, max |dT| per problem:", dict(zip([f"<{e:g}" for e in edges[1:]], hist.tolist())))
    assert max(errs) < bound, errs
    # Ground truth (motions of up to 1 m per axis and 0.1 rad): on these sparse targets (0.15 m voxels, about 2 points
    # per m^2) point-to-point converges slowly along the walls; after 100 iterations the fits measured 0.005-0.025 rad
    # and 0.05-0.6 m from the truth over seeds 0-7.
    print("ground truth: rotation error", np.round(rot, 4), "translation error", np.round(tr, 3))
    assert max(rot) < 0.03 and max(tr) < 0.7, (rot, tr)


def test_status_codes():
    src, tgt, _ = synth.make_icp_pair3(3, n_source=400, n_target=3000)
    assert o3.icp3(src, np.zeros((0, 3)))["status"] == 6
    g = np.eye(4, dtype=np.float32)
    g[0, 0] = 1.01
    r = o3.icp3(src, tgt, g)
    assert r["status"] == 5 and (r["T"] == g).all() and r["iterations"] == 0
    assert o3.icp3(src + np.float32(100), tgt)["status"] == 1  # every source point beyond maxDist
    r = o3.icp3(src + np.float32(100), tgt, params=IcpParams(trim_ratio=-1.0))
    assert r["status"] == 2
    r = o3.icp3(src, tgt, params=IcpParams(max_iterations=1))
    assert r["status"] == 0 and r["iterations"] == 1 and r["inliers"] > 0
    r = o3.icp3(src, tgt, params=IcpParams(smooth_length=0, max_iterations=7))
    assert r["status"] == 0 and r["iterations"] == 7
    r = o3.icp3(src, tgt, params=IcpParams(smooth_length=15))
    assert r["status"] == 0 and r["iterations"] >= 15
    r = o3.icp3(np.full((10, 3), np.nan, np.float32), tgt)
    assert r["status"] == 1


def test_planar_clouds_keep_z_and_match_the_2d_oracle():
    for seed in range(6):
        s2, t2, _ = synth.make_icp_pair(seed)
        r2 = orc.icp(s2, t2)
        r3 = o3.icp3(np.c_[s2, np.zeros(len(s2))], np.c_[t2, np.zeros(len(t2))])
        assert r2["status"] == r3["status"] == 0
        T = r3["T"]
        assert (T[2] == [0, 0, 1, 0]).all() and (T[:, 2] == [0, 0, 1, 0]).all() and T[2, 3] == 0
        # the xy block: the closed form and the SVD round differently
        assert np.abs(T[:2][:, [0, 1, 3]] - r2["T"][:2]).max() < 1e-4
    # A mirrored source: the 2-D cross-covariance has a negative determinant, U V^T is a reflection, and the fix turns
    # it into a proper rotation that flips z (libpointmatcher's 3-D behaviour); the 2-D closed form stays in the plane.
    # (points 1 m apart along x, within 0.1 m of the x axis: every mirrored point's nearest neighbour is its original)
    rng = np.random.default_rng(4)
    t2 = np.c_[np.arange(-20.0, 20.0), rng.uniform(-0.1, 0.1, 40)].astype(np.float32)
    s2 = t2 * np.float32([1, -1])
    r3 = o3.icp3(np.c_[s2, np.zeros(len(s2))], np.c_[t2, np.zeros(len(t2))], params=IcpParams(max_iterations=1))
    R = r3["T"][:3, :3].astype(np.float64)
    assert r3["status"] == 0 and R[2, 2] == -1 and abs(np.linalg.det(R) - 1) < 1e-5


def test_pcl_icp_rejects_before_any_device_work(tmp_path):
    icp = pcl.ICP()
    icp.params = pcl._lib.IcpParams()
    src3, tgt3 = np.zeros((5, 3), np.float32), np.zeros((6, 3), np.float32)
    with pytest.raises(TypeError):
        icp.compute(src3, np.zeros((6, 2), np.float32), np.eye(4))
    with pytest.raises(TypeError):
        icp.compute_pairs([src3], [np.zeros((6, 2), np.float32)], [[np.eye(4)]])
    with pytest.raises(ValueError):
        icp.compute(src3, tgt3, np.eye(3))
    with pytest.raises(ValueError):
        icp.compute_batch(src3, tgt3, np.zeros((2, 3, 4)))
    with pytest.raises(ValueError):
        icp.compute_pairs([src3], [tgt3], [np.zeros((1, 3, 3))])
    base = ("matcher:\n  KDTreeMatcher:\n    maxDist: 10.0\n"
            "outlierFilters:\n  - TrimmedDistOutlierFilter:\n      ratio: 0.8\n")
    yamls = {
        "plane": base + ("referenceDataPointsFilters:\n  - SurfaceNormalDataPointsFilter:\n      knn: 5\n"
                         "errorMinimizer:\n  PointToPlaneErrorMinimizer\n"),
        "data": base + "readingDataPointsFilters:\n  - MaxDistDataPointsFilter:\n      maxDist: 20.0\n",
        "mindist": base.replace("outlierFilters:\n", "outlierFilters:\n  - MinDistOutlierFilter:\n      minDist: 0.1\n"),
        "median": base.replace("outlierFilters:\n", "outlierFilters:\n  - MedianDistOutlierFilter:\n      factor: 3.0\n"),
    }
    for name, text in yamls.items():
        path = tmp_path / f"{name}.yaml"
        path.write_text(text)
        icp = pcl.ICP()
        icp.loadFromYaml(str(path))
        for call in (lambda: icp.compute(src3, tgt3, np.eye(4)), lambda: icp.compute_batch(src3, tgt3, [np.eye(4)]),
                     lambda: icp.compute_pairs([src3], [tgt3], [[np.eye(4)]])):
            with pytest.raises(NotImplementedError):
                call()
    icp.params = pcl._lib.IcpParams(flags=2)
    with pytest.raises(NotImplementedError):
        icp.compute(src3, tgt3, np.eye(4))
