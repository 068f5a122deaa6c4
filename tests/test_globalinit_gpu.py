"""GPU: global-initialisation cost (include/sonarfe.h sfe_costmap_*; reference slam.py:461-570, 683-701) against
the reference-generated fixture and the CPU oracle, through the C ABI."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import globalinit_ref as gref  # noqa: E402  (checker only)

GOLD = os.path.join(os.path.dirname(__file__), "golden", "globalinit.npz")


@pytest.fixture(scope="module")
def slam_mod():
    from sonar_slam_b200.bruce_slam import slam
    return slam


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def _row(pose):
    T = pose.matrix().astype(np.float32)
    return [T[0, 0], T[0, 1], T[1, 0], T[1, 1], T[0, 2], T[1, 2]]


def test_reference_fixture_grid_and_costs(slam_mod, gold):
    s = slam_mod.SLAM()
    sp, tp = slam_mod.Pose2(*gold["source_pose"]), slam_mod.Pose2(*gold["target_pose"])
    sub, samples = s.get_matching_cost_subroutine1(gold["source"], sp, gold["target"], tp, np.eye(3))
    grid = sub.costmap.grid()
    want = np.unpackbits(gold["grid_packed"])[: grid.size].reshape(tuple(gold["grid_shape"]))
    assert grid.shape == want.shape
    assert np.array_equal(grid, want * 255)
    costs = np.array([sub(x) for x in gold["xs"]])
    assert np.array_equal(costs, gold["costs"])
    assert np.allclose(np.array(samples), gold["pose_samples"], rtol=0, atol=1e-12)
    assert np.array_equal(sub.batch(gold["xs"], log=False), gold["costs"])
    assert len(samples) == len(gold["xs"])


def test_requires_covariance_like_reference(slam_mod, gold):
    s = slam_mod.SLAM()
    with pytest.raises(Exception):  # np.linalg.inv(None), slam.py:539
        s.get_matching_cost_subroutine1(gold["source"], slam_mod.Pose2(), gold["target"], slam_mod.Pose2())


@pytest.mark.parametrize("seed,ns,nt,K", [(0, 2000, 20000, 1), (1, 2000, 20000, 37), (2, 300, 1500, 700),
                                           (3, 1, 50, 5), (4, 5000, 3000, 6000), (5, 64, 64, 1200)])
def test_against_oracle(seed, ns, nt, K):
    from sonar_slam_b200 import _lib, synth
    rng = np.random.default_rng(seed)
    src, tgt, _ = synth.make_icp_pair(seed, n_source=max(ns, 16), n_target=max(nt, 64))
    src, tgt = src[:ns].copy(), tgt[:nt].copy()
    grid, xmin, ymin, res, hs = gref.target_grid(tgt, 0.5)
    cm = _lib.CostMap(_lib.default_context(), tgt, xmin, ymin, res, grid.shape[0], grid.shape[1], hs)
    assert np.array_equal(cm.grid(), grid)
    cm.set_source(src)
    poses = [gref.Pose2(*(rng.uniform(-1, 1, 3) * [2.0, 2.0, 0.3])) for _ in range(K)]
    if K > 4:
        poses[1] = gref.Pose2(500.0, 0.0, 0.0)  # everything outside the grid
        poses[2] = gref.Pose2(float("nan"), 0.0, 0.0)
    got = cm.score(np.array([_row(p) for p in poses], np.float32))
    check = range(K) if K <= 64 else list(range(8)) + list(rng.integers(0, K, 40))
    blas_differs = 0
    for k in check:
        # integer work: EXACT against the cost with the float32 rounding spelled out (no slack) ...
        want = gref.cost_of_transform(grid, xmin, ymin, res, src, poses[k], explicit=True)
        assert int(got[k]) == want, (k, int(got[k]), want)
        # ... which is what numpy's own float32 dot gives on this host (pinned on the reference-run fixture in
        # tests/test_oracle_globalinit.py); counted here, since a BLAS kernel without FMA may round differently
        blas_differs += int(gref.cost_of_transform(grid, xmin, ymin, res, src, poses[k]) != want)
    print("poses where numpy's dot differs from the explicit float32 formula:", blas_differs, "of", len(check))
    assert got.min() >= -ns and got.max() <= 0
    if K > 4:
        assert got[1] == 0 and got[2] == 0


def test_empty_source_and_single_target():
    from sonar_slam_b200 import _lib
    tgt = np.array([[1.0, 2.0]], np.float32)
    grid, xmin, ymin, res, hs = gref.target_grid(tgt, 0.5)
    cm = _lib.CostMap(_lib.default_context(), tgt, xmin, ymin, res, grid.shape[0], grid.shape[1], hs)
    assert np.array_equal(cm.grid(), grid)  # one ellipse, clipped by nothing
    cm.set_source(np.zeros((0, 2), np.float32))
    assert np.array_equal(cm.score(np.array([[1, 0, 0, 1, 0, 0]], np.float32)), [0])
    cm.set_source(np.array([[1.0, 2.0], [1.3, 2.0], [1.6, 2.0]], np.float32))
    assert np.array_equal(cm.score(np.array([[1, 0, 0, 1, 0, 0]], np.float32)), [-2])


def test_dense_global_initialization_finds_the_offset(slam_mod):
    """One dense Sobol batch (4096 poses, one launch) lands next to the ground-truth displacement."""
    from sonar_slam_b200 import synth
    src, tgt, T_gt = synth.make_icp_pair(21, outlier_frac=0.1)
    s = slam_mod.SLAM()
    bounds = np.array([[-1.5, 1.5], [-1.5, 1.5], [-0.15, 0.15]])
    out = s.global_initialization(src, slam_mod.Pose2(), tgt, slam_mod.Pose2(), np.eye(3), bounds, dense=4096)
    gt = np.array([T_gt[0, 2], T_gt[1, 2], np.arctan2(T_gt[1, 0], T_gt[0, 0])])
    assert out["success"] and out["fun"] <= -0.6 * len(src)
    assert np.all(np.abs(out["x"] - gt) < [0.5, 0.5, 0.06]), (out["x"], gt)
    # the reference's own optimiser on the same (GPU-evaluated) function reaches a cost no better than the dense batch
    ref = s.global_initialization(src, slam_mod.Pose2(), tgt, slam_mod.Pose2(), np.eye(3), bounds,
                                  initialization_params=(50, 1, 0.01))
    assert ref["success"] and ref["fun"] >= out["fun"] - 1e-9
