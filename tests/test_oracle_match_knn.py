"""CPU: the k-nearest-neighbour oracle (oracle/knn_ref.c orc_match_knn) against independent statements of the rule --
scipy's cKDTree on tie-free clouds, and a numpy lexsort over (float32 squared distance, index) on lattices and
duplicate points, where ties decide the order."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import knn_ref, oracle as orc


def _lexsort_knn(ref, pts, knn, max_dist):
    """For every query: the accepted points (float32 d2 = dx*dx + dy*dy <= max_dist^2, finite) sorted by (d2, index)."""
    ref, pts = np.asarray(ref, np.float32), np.asarray(pts, np.float32)
    max_d2 = np.float32(max_dist) * np.float32(max_dist)
    ids = np.full((knn, len(pts)), -1, np.int32)
    d = np.full((knn, len(pts)), np.inf, np.float32)
    for i, q in enumerate(pts):
        dx, dy = q[0] - ref[:, 0], q[1] - ref[:, 1]
        d2 = dx * dx + dy * dy
        ok = np.nonzero((d2 <= max_d2) & np.isfinite(d2))[0]
        order = ok[np.lexsort((ok, d2[ok]))][:knn]
        ids[:len(order), i] = order
        d[:len(order), i] = d2[order]
    return ids, d


@pytest.mark.parametrize("knn", [2, 3, 5, 16])
def test_equals_ckdtree_on_tie_free_clouds(knn):
    rng = np.random.default_rng(knn)
    ref = rng.uniform(0, 40, (3000, 2)).astype(np.float32)
    pts = rng.uniform(-5, 45, (400, 2)).astype(np.float32)
    for max_dist in (1.5, np.inf):
        ids, d = knn_ref.match_knn(ref, pts, knn, max_dist)
        want_d, want_i = cKDTree(ref.astype(np.float64)).query(pts.astype(np.float64), k=knn,
                                                               distance_upper_bound=max_dist)
        want_i = np.where(want_i == len(ref), -1, want_i).T
        assert np.array_equal(ids, want_i), (knn, max_dist)
        hit = ids >= 0
        assert np.allclose(d[hit], (want_d.T[hit] ** 2), rtol=1e-5)
        assert np.isinf(d[~hit]).all()
        assert hit.any() and (max_dist == np.inf or (~hit).any())


@pytest.mark.parametrize("knn", [2, 5, 16])
def test_ties_follow_the_lower_index_on_lattices_and_duplicates(knn):
    rng = np.random.default_rng(40 + knn)
    g = np.arange(12, dtype=np.float32)
    lattice = np.stack(np.meshgrid(g, g), -1).reshape(-1, 2)[rng.permutation(144)]
    dup = np.concatenate([lattice[:50], lattice[:50][::-1], lattice[10:20]])      # every point two or three times
    q_lat = np.concatenate([lattice[::7], lattice[::5] + np.float32(0.5), np.float32([[5.5, 5.5], [-3, -3]])])
    for ref in (lattice, dup):
        for max_dist in (0.0, 1.0, 2.5, np.inf):
            ids, d = knn_ref.match_knn(ref, q_lat, knn, max_dist)
            wi, wd = _lexsort_knn(ref, q_lat, knn, max_dist)
            assert np.array_equal(ids, wi), (knn, max_dist)
            assert np.array_equal(d.view(np.uint32), wd.view(np.uint32))


def test_row_zero_is_the_nearest_neighbour_and_rows_are_prefixes():
    rng = np.random.default_rng(7)
    ref = np.round(rng.uniform(0, 20, (800, 2)) * 2).astype(np.float32) / 2          # many exact ties
    pts = np.concatenate([rng.uniform(-2, 22, (300, 2)), [[np.nan, 1.0], [np.nan, np.nan]]]).astype(np.float32)
    for max_dist in (0.0, 0.7, 3.0, np.inf):
        one = orc.match(ref, pts, max_dist, brute=True)
        ids16, d16 = knn_ref.match_knn(ref, pts, 16, max_dist)
        assert np.array_equal(ids16[:1], one[0]) and np.array_equal(d16[:1], one[1])
        for k in (2, 5, 9):
            ik, dk = knn_ref.match_knn(ref, pts, k, max_dist)
            assert np.array_equal(ik, ids16[:k]) and np.array_equal(dk, d16[:k])
        assert (ids16[:, -2:] == -1).all()                                            # NaN queries: unmatched
    empty = knn_ref.match_knn(np.zeros((0, 2), np.float32), pts, 4, 1.0)
    assert (empty[0] == -1).all() and np.isinf(empty[1]).all()
    few = knn_ref.match_knn(ref[:3], pts[:10], 5, np.inf)                                 # knn above the reference size
    assert (np.sort(few[0][:3], 0) == np.arange(3)[:, None]).all() and (few[0][3:] == -1).all()
