"""CPU: SurfaceNormalDataPointsFilter and ShadowDataPointsFilter on the reading cloud in icp.yaml -- the parser's accept /
refuse table, and the oracle (oracle/shadow_ref.c) against independent statements: the reading normals against a NumPy
brute force, the shadow test against a literal float32 Python statement, a chain against its steps composed, and one
ICP iteration on pre-filtered clouds against the oracle without reading filters."""
import ctypes
import ctypes.util

import numpy as np
import pytest

from oracle import oracle as orc
from oracle import sampling_normal_ref as snr
from oracle import shadow_ref as shr
from sonar_slam_b200 import _lib, synth
from sonar_slam_b200.bruce_slam import pcl

F32 = np.float32
NRM, SHD = "SurfaceNormalDataPointsFilter", "ShadowDataPointsFilter"
MAXD, MIND = "MaxDistDataPointsFilter: {maxDist: 20.0}", "MinDistDataPointsFilter: {minDist: 0.5}"


def _yaml(reading=(), reference=(), minimizer="PointToPointErrorMinimizer"):
    def chain(fs):
        return "".join(f"  - {f}\n" for f in fs) or "  []\n"
    return (f"readingDataPointsFilters:\n{chain(reading)}referenceDataPointsFilters:\n{chain(reference)}"
            f"matcher:\n  KDTreeMatcher:\n    maxDist: 10.0\nerrorMinimizer:\n  {minimizer}\n")


# ---------------------------------------------------------------- the parser
def test_accepted_chains():
    cfg = pcl.parse_icp_yaml(_yaml([MAXD, f"{NRM}: {{knn: 7}}", f"{SHD}: {{eps: 0.2}}", MIND]))
    assert cfg.filters.data_filters("reading") == [(_lib.MAX_DIST, -1, 20.0), (_lib.NORMALS, 7, 0.0),
                                                   (_lib.SHADOW, 0, F32(0.2)), (_lib.MIN_DIST, -1, 0.5)]
    # upstream defaults: knn 5, eps 0.1
    cfg = pcl.parse_icp_yaml(_yaml([NRM, SHD]))
    assert cfg.filters.data_filters("reading") == [(_lib.NORMALS, 5, 0.0), (_lib.SHADOW, 0, F32(0.1))]
    # down-samplers before the normals; the normals alone; knn 3 and 16; eps 0, negative and large
    cfg = pcl.parse_icp_yaml(_yaml(["VoxelGridDataPointsFilter: {vSizeX: 0.2, vSizeY: 0.2}",
                                    "OctreeGridDataPointsFilter: {maxSizeByNode: 0.3}", f"{NRM}: {{knn: 16}}",
                                    f"{SHD}: {{eps: -0.3}}"]))
    assert [f[0] for f in cfg.filters.data_filters("reading")] == [_lib.VOXEL, _lib.OCTREE, _lib.NORMALS, _lib.SHADOW]
    for eps in (0, 2.5):
        cfg = pcl.parse_icp_yaml(_yaml([f"{NRM}: {{knn: 3}}", f"{SHD}: {{eps: {eps}}}"]))
        assert cfg.filters.data_filters("reading")[1] == (_lib.SHADOW, 0, F32(eps))
    assert pcl.parse_icp_yaml(_yaml([NRM])).filters.data_filters("reading") == [(_lib.NORMALS, 5, 0.0)]
    # keepNormals 0 is a no-op; the reading normals next to point-to-plane's reference normals
    assert pcl.parse_icp_yaml(_yaml([f"{NRM}: {{keepNormals: 0}}", MAXD])).filters.data_filters("reading") == \
        [(_lib.MAX_DIST, -1, 20.0)]
    cfg = pcl.parse_icp_yaml(_yaml([NRM, SHD], [f"{NRM}: {{knn: 9}}"], "PointToPlaneErrorMinimizer"))
    assert cfg.minimizer == 1 and cfg.normals_knn == 9 and cfg.filters.data_filters("reference") == []


@pytest.mark.parametrize("reading, reference, exc, match", [
    ([SHD], [], ValueError, "normals"),
    ([f"{NRM}: {{keepNormals: 0}}", SHD], [], ValueError, "normals"),
    ([SHD, NRM], [], ValueError, "normals"),
    ([NRM, f"{SHD}: {{eps: .nan}}"], [], ValueError, "eps"),
    ([NRM, f"{SHD}: {{eps: .inf}}"], [], ValueError, "eps"),
    ([f"{NRM}: {{knn: 2}}"], [], NotImplementedError, "knn"),
    ([f"{NRM}: {{knn: 17}}"], [], NotImplementedError, "knn"),
    ([f"{NRM}: {{knn: 4.5}}"], [], NotImplementedError, "knn"),
    ([f"{NRM}: {{epsilon: 0.5}}"], [], NotImplementedError, "epsilon"),
    ([NRM, NRM], [], NotImplementedError, "second"),
    ([NRM, SHD, NRM], [], NotImplementedError, "second"),
    ([NRM, "OctreeGridDataPointsFilter: {maxSizeByNode: 0.3}"], [], NotImplementedError, f"after {NRM}"),
    ([NRM, "VoxelGridDataPointsFilter: {vSizeX: 0.2, vSizeY: 0.2}"], [], NotImplementedError, f"after {NRM}"),
    ([NRM, "SamplingSurfaceNormalDataPointsFilter: {samplingMethod: 1}"], [], NotImplementedError,
     "reading filter SamplingSurfaceNormalDataPointsFilter"),
    ([], [NRM, SHD], NotImplementedError, SHD),
    ([], [SHD], NotImplementedError, SHD),
    ([MAXD, MIND, "MaxDistDataPointsFilter: {dim: 0, maxDist: 9}", NRM, SHD], [], NotImplementedError, "more than 4"),
    ([MAXD, MIND, NRM, SHD, "MinDistDataPointsFilter: {dim: 1, minDist: 1}"], [], NotImplementedError, "more than 4"),
])
def test_refusals(reading, reference, exc, match):
    with pytest.raises(exc, match=match):
        pcl.parse_icp_yaml(_yaml(reading, reference))


def test_three_column_clouds_stay_refused():
    icp = pcl.ICP()
    icp.params = pcl.parse_icp_yaml(_yaml([NRM, SHD]))
    with pytest.raises(NotImplementedError, match="3-column"):
        icp.compute(np.zeros((10, 3), F32), np.zeros((10, 3), F32), np.eye(4, dtype=F32))


# ---------------------------------------------------------------- the reading normals against a NumPy brute force
def _np_normal(q):
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
        return F32(0), F32(0)
    d = F32(F32(0.5) * F32(a - c))
    r = np.sqrt(F32(F32(d * d) + F32(b * b)), dtype=F32)
    if r == 0:
        return F32(1), F32(0)
    ux, uy = (F32(r + d), b) if d >= 0 else (b, F32(r - d))
    ln = np.sqrt(F32(F32(ux * ux) + F32(uy * uy)), dtype=F32)
    return F32(-F32(uy / ln)), F32(ux / ln)


def _np_reading_normals(pts, knn):
    pts = np.asarray(pts, F32).reshape(-1, 2)
    n = len(pts)
    out = np.zeros((n, 2), F32)
    if n == 0:
        return out
    sx, sy = F32(0), F32(0)
    for x, y in pts:
        sx, sy = F32(sx + x), F32(sy + y)
    c = pts - np.array([F32(sx / F32(n)), F32(sy / F32(n))], F32)
    for i in range(n):
        d = c - c[i]
        d2 = (d[:, 0] * d[:, 0]) + (d[:, 1] * d[:, 1])  # float32, each operation rounded
        nb = np.lexsort((np.arange(n), d2))[:knn]      # ascending distance, ties to the lower index
        out[i] = _np_normal(c[nb])
    return out


def _normal_clouds():
    rng = np.random.default_rng(7)
    lattice = (np.stack(np.meshgrid(np.arange(9), np.arange(7)), -1).reshape(-1, 2) * F32(0.25)).astype(F32)
    ring = np.stack([np.cos(np.arange(12) * np.pi / 6), np.sin(np.arange(12) * np.pi / 6)], -1).astype(F32) * 3
    return {
        "empty": np.zeros((0, 2), F32),
        "one": np.array([[1.5, -2.0]], F32),
        "two": np.array([[1.0, 1.0], [2.0, 3.0]], F32),
        "coincident": np.tile(np.array([[0.5, -0.5]], F32), (20, 1)),
        "coincident_pairs": np.repeat(rng.normal(0, 3, (15, 2)).astype(F32), 2, axis=0),
        "collinear": np.stack([np.linspace(-4, 4, 25), np.linspace(1, 3, 25)], -1).astype(F32),
        "equidistant": np.concatenate([np.zeros((1, 2), F32), ring, lattice]),
        "lattice": lattice[rng.permutation(len(lattice))],
        "random": rng.normal(5, 4, (150, 2)).astype(F32),
        "scan": synth.make_icp_pair(3, n_source=200, n_target=300)[0],
    }


@pytest.mark.parametrize("knn", [3, 5, 16])
@pytest.mark.parametrize("cloud", list(_normal_clouds()))
def test_reading_normals_equal_numpy_bit_for_bit(cloud, knn):
    pts = _normal_clouds()[cloud]
    got, want = shr.reading_normals(pts, knn), _np_reading_normals(pts, knn)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (cloud, knn)


def test_clouds_smaller_than_knn():
    for n in range(1, 6):
        pts = np.random.default_rng(n).normal(0, 1, (n, 2)).astype(F32)
        got, want = shr.reading_normals(pts, 16), _np_reading_normals(pts, 16)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), n


# ---------------------------------------------------------------- the shadow test against a literal statement
_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.sinf.restype, _libm.sinf.argtypes = ctypes.c_float, [ctypes.c_float]


def _py_shadow(x, y, nx, ny, eps):
    """keep iff |n^ . p^| > sinf(eps), Eigen's normalized() on both, float32 operation by operation"""
    def unit(a, b):
        s = F32(F32(a * a) + F32(b * b))
        if s > 0:
            ln = np.sqrt(s, dtype=F32)
            return F32(a / ln), F32(b / ln)
        return a, b
    with np.errstate(over="ignore"):  # (a squared norm may overflow to +inf, as in C)
        nx, ny = unit(F32(nx), F32(ny))
        px, py = unit(F32(x), F32(y))
    return bool(abs(F32(F32(nx * px) + F32(ny * py))) > F32(_libm.sinf(F32(eps))))


def test_sin_eps_is_the_c_librarys():
    for eps in (0.0, 0.1, -0.3, 1.0, 2.5, 100.0):
        assert shr.sin_eps(eps).view(np.uint32) == F32(_libm.sinf(F32(eps))).view(np.uint32)


def test_shadow_keep_equals_the_literal_statement():
    rng = np.random.default_rng(3)
    special = [(0, 0, 1, 0), (0, 0, 0, 0), (3, 4, 0, 0), (1, 0, 0, 1), (1, 0, 1, 0), (-2, 0, 1, 0), (1, 1, 1, -1),
               (1e-20, 0, 0, 1e-20), (1e20, 1e20, -1, 1), (5, 0, F32(np.cos(F32(1.4708))), F32(np.sin(F32(1.4708))))]
    cases = special + [tuple(v) for v in rng.normal(0, 3, (400, 4)).astype(F32)]
    for eps in (0.0, 0.1, -0.2, 1.2, 2.0, 10.0, 0.0998):
        for x, y, nx, ny in cases:
            assert shr.shadow_keep(x, y, nx, ny, eps) == _py_shadow(x, y, nx, ny, eps), (x, y, nx, ny, eps)
    # a point at the origin and a zero normal: the dot is 0, kept only for a negative threshold
    assert not shr.shadow_keep(0, 0, 1, 0, 0.0) and shr.shadow_keep(0, 0, 1, 0, -0.1)
    assert not shr.shadow_keep(3, 4, 0, 0, 0.0) and shr.shadow_keep(3, 4, 0, 0, -0.1)
    # a wall seen head-on is kept, a streak along the ray is not
    assert shr.shadow_keep(10, 0, 1, 0, 0.1) and not shr.shadow_keep(10, 0, 0, 1, 0.1)


# ---------------------------------------------------------------- a chain against its steps composed
def test_chain_equals_its_steps():
    from oracle import icp_filters_ref as fr
    s, _, _ = synth.make_icp_pair(21, n_source=900, n_target=100)
    s = (s + F32(3.0)).astype(F32)
    for knn, eps in ((3, 0.1), (5, 0.3), (16, -0.1), (7, 0.0)):
        chain = [(_lib.MAX_DIST, -1, 25.0), (_lib.NORMALS, knn, 0.0), (_lib.SHADOW, 0, eps), (_lib.MIN_DIST, -1, 2.0)]
        got = shr.data_filters(s, chain)
        a = fr.data_filters(s, [chain[0]])
        n = shr.reading_normals(a, knn)
        keep = np.array([_py_shadow(x, y, nx, ny, eps) for (x, y), (nx, ny) in zip(a, n)], bool)
        want = fr.data_filters(a[keep], [chain[3]])
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (knn, eps)
        assert 0 < len(got) < len(s)
    # the normals alone change nothing; a shadow right after them: the same as the composed filter
    assert np.array_equal(shr.data_filters(s, [(_lib.NORMALS, 5, 0.0)]), s)


def test_one_iteration_on_prefiltered_clouds_equals_the_oracle():
    for minimizer in (0, 1):
        prm = orc.IcpParams(minimizer=minimizer, normals_knn=5, max_iterations=1, smooth_length=0)
        for seed in (1, 2, 3):
            s, t, g = synth.make_icp_pair(seed, n_source=500, n_target=900)
            chain = [(_lib.NORMALS, 5, 0.0), (_lib.SHADOW, 0, 0.15)]
            got = shr.icp(s, t, g.astype(F32), prm, shr.IcpFilters(reading=chain))
            want = snr.icp(shr.data_filters(s, chain), t, g.astype(F32), prm)
            assert (got["status"], got["iterations"], got["inliers"]) == \
                (want["status"], want["iterations"], want["inliers"]), (minimizer, seed)
            assert np.array_equal(got["T"].view(np.uint32), want["T"].view(np.uint32)), (minimizer, seed)
            assert got["iterations"] == 1 and got["inliers"] < len(s)
