"""CPU: SamplingSurfaceNormalDataPointsFilter in icp.yaml -- the parser's accept / refuse table, and the oracle filter
(oracle/sampling_normal_ref.c) against an independent NumPy recursion with np.lexsort splits, point for point and bit
for bit."""
import numpy as np
import pytest

from oracle import sampling_normal_ref as snr
from sonar_slam_b200 import _lib
from sonar_slam_b200.bruce_slam import pcl

F32 = np.float32
SN = "SamplingSurfaceNormalDataPointsFilter"


def _yaml(ref, minimizer="PointToPlaneErrorMinimizer", reading=""):
    return (f"readingDataPointsFilters:\n{reading or '  []'}\nreferenceDataPointsFilters:\n{ref}\n"
            f"matcher:\n  KDTreeMatcher:\n    maxDist: 10.0\nerrorMinimizer:\n  {minimizer}\n")


def test_accepts_the_filter_as_the_normal_source():
    cfg = pcl.parse_icp_yaml(_yaml(f"  - MaxDistDataPointsFilter: {{maxDist: 20.0}}\n"
                                   f"  - {SN}: {{knn: 10, samplingMethod: 1, maxBoxDim: 0.5}}"))
    assert cfg.minimizer == 1 and cfg.normals_knn == 10
    assert cfg.filters.data_filters("reference") == [(_lib.MAX_DIST, -1, 20.0), (_lib.SAMPLING_NORMALS, 1, 0.5)]
    cfg = pcl.parse_icp_yaml(_yaml(f"  - {SN}: {{knn: 64, samplingMethod: 0, ratio: 1}}"))
    assert cfg.normals_knn == 64 and cfg.filters.data_filters("reference") == [(_lib.SAMPLING_NORMALS, 0, np.inf)]
    # a plain down-sampler for point-to-point, also without normals
    cfg = pcl.parse_icp_yaml(_yaml(f"  - {SN}: {{knn: 3, samplingMethod: 1, keepNormals: 0}}",
                                   "PointToPointErrorMinimizer"))
    assert cfg.minimizer == 0 and cfg.normals_knn == 3


@pytest.mark.parametrize("ref, exc, match", [
    (f"  - {SN}: {{samplingMethod: 1, keepNormals: 0}}", ValueError, "normals"),
    (f"  - {SN}: {{samplingMethod: 1}}\n  - MaxDistDataPointsFilter: {{maxDist: 5.0}}", NotImplementedError,
     "SurfaceNormalDataPointsFilter"),
    (f"  - {SN}: {{samplingMethod: 1}}\n  - VoxelGridDataPointsFilter: {{vSizeX: 1, vSizeY: 1}}", NotImplementedError,
     "SurfaceNormalDataPointsFilter"),
    (f"  - {SN}: {{samplingMethod: 1}}\n  - SurfaceNormalDataPointsFilter: {{knn: 5}}", NotImplementedError,
     "one source of normals"),
    (f"  - SurfaceNormalDataPointsFilter: {{knn: 5}}\n  - {SN}: {{samplingMethod: 1}}", NotImplementedError,
     "one source of normals"),
    (f"  - {SN}: {{samplingMethod: 1}}\n  - {SN}: {{samplingMethod: 1}}", NotImplementedError, "one source of normals"),
    (f"  - {SN}: {{knn: 2, samplingMethod: 1}}", NotImplementedError, "knn"),
    (f"  - {SN}: {{knn: 65, samplingMethod: 1}}", NotImplementedError, "knn"),
    (f"  - {SN}: {{knn: 7.5, samplingMethod: 1}}", NotImplementedError, "knn"),
    (f"  - {SN}: {{samplingMethod: 0}}", NotImplementedError, "random"),
    (f"  - {SN}: {{samplingMethod: 0, ratio: 0.7}}", NotImplementedError, "random"),
    (f"  - {SN}: {{samplingMethod: 1, ratio: 0}}", ValueError, "ratio"),
    (f"  - {SN}: {{samplingMethod: 1, ratio: 1.5}}", ValueError, "ratio"),
    (f"  - {SN}: {{samplingMethod: 1, maxBoxDim: .nan}}", ValueError, "maxBoxDim"),
    (f"  - {SN}: {{samplingMethod: 1, maxBoxDim: -1}}", ValueError, "maxBoxDim"),
    (f"  - {SN}: {{samplingMethod: 2}}", ValueError, "samplingMethod"),
    ("".join(f"  - MaxDistDataPointsFilter: {{maxDist: {20 + k}.0}}\n" for k in range(4)) + f"  - {SN}: {{samplingMethod: 1}}",
     NotImplementedError, "more than 4"),
])
def test_refusals(ref, exc, match):
    with pytest.raises(exc, match=match):
        pcl.parse_icp_yaml(_yaml(ref))


def test_reading_side_is_refused():
    with pytest.raises(NotImplementedError, match=f"reading filter {SN}"):
        pcl.parse_icp_yaml(_yaml("  []", reading=f"  - {SN}: {{samplingMethod: 1}}"))


# ---------------------------------------------------------------- the oracle against an independent recursion
def _normal(q):
    """orc_surface_normals' closed form on the rows of q, float32 operation by operation"""
    k = F32(len(q))
    sx, sy = F32(0), F32(0)
    for x, y in q:
        sx, sy = F32(sx + x), F32(sy + y)
    mx, my = F32(sx / k), F32(sy / k)
    a = b = c = F32(0)
    for x, y in q:
        ux, uy = F32(x - mx), F32(y - my)
        a, b, c = F32(a + F32(ux * ux)), F32(b + F32(ux * uy)), F32(c + F32(uy * uy))
    a, b, c = F32(a / k), F32(b / k), F32(c / k)
    if a == 0 and b == 0 and c == 0:
        return (mx, my), (F32(0), F32(0))
    d = F32(F32(0.5) * F32(a - c))
    r = np.sqrt(F32(F32(d * d) + F32(b * b)), dtype=F32)
    if r == 0:
        return (mx, my), (F32(1), F32(0))
    ux, uy = (F32(r + d), b) if d >= 0 else (b, F32(r - d))
    ln = np.sqrt(F32(F32(ux * ux) + F32(uy * uy)), dtype=F32)
    return (mx, my), (F32(-F32(uy / ln)), F32(ux / ln))


def _numpy_filter(pts, knn, method, max_box):
    pts = pts.astype(F32)
    keep, val, nrm = {}, {}, {}

    def build(idx, mn, mx):
        if len(idx) <= knn:
            if len(idx):
                fuse(np.sort(idx))
            return
        d = 1 if F32(mx[1] - mn[1]) > F32(mx[0] - mn[0]) else 0
        coord = pts[idx, d] + F32(0)  # -0 orders as +0
        idx = idx[np.lexsort((idx, coord))]
        left = len(idx) - len(idx) // 2
        cut = pts[idx[left], d]
        lmx, rmn = mx.copy(), mn.copy()
        lmx[d], rmn[d] = cut, cut
        build(idx[:left], mn, lmx)
        build(idx[left:], rmn, mx)

    def fuse(idx):
        q = pts[idx]
        ext = q.max(0) - q.min(0)
        if max(ext[0], ext[1]) > F32(max_box):
            return
        c, n = _normal(q)
        for j, i in enumerate(idx[:1] if method == 1 else idx):
            keep[i] = True
            val[i] = c if method == 1 else tuple(pts[i])
            nrm[i] = n

    if len(pts):
        build(np.arange(len(pts)), pts.min(0), pts.max(0))
    order = sorted(keep)
    return (np.array([val[i] for i in order], F32).reshape(-1, 2), np.array([nrm[i] for i in order], F32).reshape(-1, 2))


def _clouds():
    rng = np.random.default_rng(7)
    lattice = (np.stack(np.meshgrid(np.arange(23), np.arange(17)), -1).reshape(-1, 2) * 0.25).astype(F32)
    lattice = lattice[rng.permutation(len(lattice))]
    walls = np.concatenate([np.stack([np.linspace(0, 9, 200), np.full(200, 3.0)], 1),
                            np.stack([np.full(150, -2.0), np.linspace(-4, 4, 150)], 1)]).astype(F32)
    return {
        "random": rng.normal(0, 5, (700, 2)).astype(F32),
        "lattice_ties": np.concatenate([lattice, lattice[:90], -lattice[:40]]),
        "walls": walls[rng.permutation(len(walls))],
        "coincident": np.tile(np.array([[1.5, -2.0]], F32), (50, 1)),
        "signed_zero": np.array([[0.0, 1.0], [-0.0, 2.0], [0.0, -0.0], [-0.0, 0.0], [1.0, -0.0]] * 4, F32),
        "single": np.array([[3.0, 4.0]], F32),
        "root_box": rng.normal(0, 1, (3, 2)).astype(F32),
        "empty": np.zeros((0, 2), F32),
    }


@pytest.mark.parametrize("max_box", [np.inf, 0.6, 0.0])
@pytest.mark.parametrize("method", [0, 1])
@pytest.mark.parametrize("knn", [3, 7, 64])
@pytest.mark.parametrize("name", list(_clouds()))
def test_oracle_equals_the_numpy_recursion(name, knn, method, max_box):
    pts = _clouds()[name]
    got_p, got_n = snr.sampling_normals(pts, knn, method, max_box)
    want_p, want_n = _numpy_filter(pts, knn, method, max_box)
    assert got_p.shape == want_p.shape
    assert np.array_equal(got_p.view(np.uint32), want_p.view(np.uint32))
    assert np.array_equal(got_n.view(np.uint32), want_n.view(np.uint32))


def test_max_box_drops_whole_boxes():
    pts = _clouds()["random"]
    full, _ = snr.sampling_normals(pts, 7, 0, np.inf)
    part, _ = snr.sampling_normals(pts, 7, 0, 0.6)
    assert len(full) == len(pts) and 0 < len(part) < len(pts)


def test_chain_and_point_to_point_down_sampler():
    """The filter after a distance filter, and point-to-point ICP with the filter equal to the ICP on the filtered
    target without it"""
    from oracle import robust_ref
    from oracle.oracle import IcpParams
    from sonar_slam_b200 import synth
    s, t, T = synth.make_icp_pair(3, n_source=300, n_target=1500)
    flt = [(_lib.MAX_DIST, -1, 25.0), (snr.SAMPLING_NORMALS, 1, np.inf)]
    pts, nrm = snr.data_filters(t, flt, knn=5)
    want, _ = snr.sampling_normals(t[np.sqrt((t * t).sum(1, dtype=F32), dtype=F32) < 25.0], 5, 1)
    assert np.array_equal(pts, want) and nrm is not None
    prm = IcpParams(normals_knn=5)
    a = snr.icp(s, t, T.astype(F32), prm, snr.IcpFilters(reference=flt))
    b = robust_ref.icp(s, pts, T.astype(F32), prm)
    assert (a["status"], a["iterations"], a["inliers"]) == (b["status"], b["iterations"], b["inliers"])
    assert np.array_equal(a["T"], b["T"])
