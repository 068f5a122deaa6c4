"""CPU-only: VoxelGridDataPointsFilter in the ICP data-filter chains.

  * parse_icp_yaml reads the module in either chain: upstream's defaults, the ignored parameters, the rejected sizes and
    useCentroid 0, the fifth data filter of a cloud, and the module after the normals filter.
  * oracle/voxel_filter_ref.c's voxel filter equals a literal statement written here (a Python loop over float32
    scalars with a dict of voxels) on lattice-aligned points, points on voxel boundaries, negative coordinates, one
    voxel holding everything and every point in its own voxel, and reports the voxel-count overflow.
  * its chains mixing voxel, octree and distance filters equal the composition of the steps, and one iteration through
    a voxel chain is the computation on the pre-filtered clouds.
"""
import numpy as np
import pytest

from oracle import octree_filter_ref as ofr
from oracle import oracle as orc
from oracle import voxel_filter_ref as vfr
from sonar_slam_b200 import _lib, synth
from sonar_slam_b200.bruce_slam import pcl
from test_icp_filters_cpu import _np_data_filters, _np_one_iteration, _yaml

F32 = np.float32
VOX = "VoxelGridDataPointsFilter"
OCT = "OctreeGridDataPointsFilter"
MAXD = "MaxDistDataPointsFilter: {dim: -1, maxDist: 25.0}"
NORMALS = "SurfaceNormalDataPointsFilter: {knn: 5}"


# ------------------------------------------------------------------------------------------ parser
def test_parser_reads_the_voxel_filter_in_either_chain():
    assert _lib.VOXEL == vfr.VOXEL == 4
    # upstream's defaults: vSizeX = vSizeY = 1, useCentroid 1
    p = pcl.parse_icp_yaml(_yaml(reading=[VOX]))
    assert p.filters.data_filters("reading") == [(_lib.VOXEL, 1, 1.0)] and p.filters.n_reference == 0
    # vSizeZ and averageExistingDescriptors are moot on 2-D clouds without descriptors
    q = f"{VOX}: {{vSizeX: 0.2, vSizeY: 0.2, vSizeZ: 3.0, useCentroid: 1, averageExistingDescriptors: 0}}"
    p = pcl.parse_icp_yaml(_yaml(reference=[q]))
    assert p.filters.data_filters("reference") == [(_lib.VOXEL, 1, pytest.approx(0.2))] and p.filters.n_reading == 0
    # mixed with the distance and octree filters, in listed order, before the normals filter
    p = pcl.parse_icp_yaml(_yaml(reading=[MAXD, f"{VOX}: {{vSizeX: 0.5, vSizeY: 0.5}}"],
                                 reference=[f"{VOX}: {{vSizeX: 0.25, vSizeY: 0.25}}", f"{OCT}: {{maxSizeByNode: 1}}",
                                            NORMALS],
                                 minimizer="PointToPlaneErrorMinimizer"))
    assert p.minimizer == 1
    assert p.filters.data_filters("reading") == [(_lib.MAX_DIST, -1, 25.0), (_lib.VOXEL, 1, 0.5)]
    assert p.filters.data_filters("reference") == [(_lib.VOXEL, 1, 0.25), (_lib.OCTREE, 0, 1.0)]
    # the same voxel filter twice is a chain, not a duplicate; four per cloud
    p = pcl.parse_icp_yaml(_yaml(reading=[VOX] * 3 + [MAXD]))
    assert p.filters.n_reading == 4


@pytest.mark.parametrize("bad", [
    f"{VOX}: {{vSizeX: 0, vSizeY: 0}}",
    f"{VOX}: {{vSizeX: -0.5, vSizeY: -0.5}}",
    f"{VOX}: {{vSizeX: .nan, vSizeY: .nan}}",
    f"{VOX}: {{vSizeX: .inf, vSizeY: .inf}}",
    f"{VOX}: {{vSizeX: 0.5, vSizeY: -.inf}}",
    f"{VOX}: {{vSizeX: 0.5, vSizeY: 0.5, useCentroid: 2}}",
])
def test_parser_rejects_bad_voxel_values(bad):
    for side in ("reading", "reference"):
        with pytest.raises(ValueError):
            pcl.parse_icp_yaml(_yaml(**{side: [bad]}))


@pytest.mark.parametrize("bad, why", [
    (f"{VOX}: {{vSizeX: 0.5, vSizeY: 0.25}}", "vSizeY"),
    (f"{VOX}: {{vSizeX: 0.5}}", "vSizeY"),  # vSizeY keeps upstream's default, 1
    (f"{VOX}: {{vSizeX: 0.5, vSizeY: 0.5, useCentroid: 0}}", "useCentroid 0"),
])
def test_parser_rejects_unimplemented_voxel_settings(bad, why):
    for side in ("reading", "reference"):
        with pytest.raises(NotImplementedError, match=why):
            pcl.parse_icp_yaml(_yaml(**{side: [bad]}))


def test_parser_rejects_a_fifth_filter_and_a_voxel_filter_after_the_normals():
    vox = f"{VOX}: {{vSizeX: 0.3, vSizeY: 0.3}}"
    with pytest.raises(NotImplementedError, match="more than 4"):
        pcl.parse_icp_yaml(_yaml(reading=[vox, MAXD, vox, f"{OCT}: {{maxSizeByNode: 0.3}}", vox]))
    with pytest.raises(NotImplementedError, match="SurfaceNormalDataPointsFilter"):
        pcl.parse_icp_yaml(_yaml(reference=[NORMALS, vox], minimizer="PointToPlaneErrorMinimizer"))
    assert pcl.parse_icp_yaml(_yaml(reference=[vox, NORMALS], minimizer="PointToPlaneErrorMinimizer")).minimizer == 1


# ------------------------------------------------------------------------------------------ oracle: the filter
def _py_voxel(pts, vsize):
    """A second, literal statement of VoxelGridDataPointsFilter (useCentroid), a Python loop over numpy float32 scalars
    with a dict from voxel index to its first point; shares no code with oracle/voxel_filter_ref.c."""
    f = np.float32
    pts = np.asarray(pts, np.float32)
    v = f(vsize)
    if len(pts) == 0:
        return np.zeros((0, 2), np.float32)
    min_b = [f(pts[:, d].min()) / v for d in range(2)]
    max_b = [f(pts[:, d].max()) / v for d in range(2)]
    num_div_x = 1 + int(np.floor(f(max_b[0] - min_b[0])))
    first, count, acc = {}, {}, {}
    for p in range(len(pts)):
        i = int(np.floor(f(pts[p, 0] / v - min_b[0])))
        j = int(np.floor(f(pts[p, 1] / v - min_b[1])))
        idx = i + j * num_div_x
        if idx not in first:
            first[idx], count[idx], acc[idx] = p, 0, [f(pts[p, 0]), f(pts[p, 1])]
        else:
            acc[idx] = [f(acc[idx][0] + pts[p, 0]), f(acc[idx][1] + pts[p, 1])]
        count[idx] += 1
    keep = sorted((first[k], k) for k in first)
    return np.array([[acc[k][0] / f(count[k]), acc[k][1] / f(count[k])] for _, k in keep], np.float32).reshape(-1, 2)


def _clouds():
    rng = np.random.default_rng(5)
    lattice = (np.round(rng.uniform(-20, 20, (1500, 2)) / 0.25) * 0.25).astype(F32)  # on every voxel boundary
    return {
        "random": (rng.uniform(-30, 30, (2500, 2)).astype(F32), 0.7),
        "sonar": (synth.make_icp_pair(3, n_source=800, n_target=4000)[1], 0.3),
        "lattice": (lattice, 0.5),
        "boundaries": (np.array([[0, 0], [1, 0], [0.999999, 1], [1, 1], [2, 2], [-1, -1], [-0.0, 1.5]], F32), 1.0),
        "negative": (rng.uniform(-50, -10, (800, 2)).astype(F32), 0.35),
        "one_voxel": (rng.uniform(3.0, 3.2, (500, 2)).astype(F32), 10.0),
        "own_voxel": (np.c_[np.arange(300) * 2.0 - 100.0, np.arange(300) % 7 * 3.0].astype(F32), 0.5),
        "single": (np.array([[7.0, -3.5]], F32), 0.2),
        # a voxel of 40 points at x = -0.0 (a zero lateral coordinate negated): its centroid keeps x = -0.0
        "negative_zero": (np.c_[np.full(40, -0.0), rng.uniform(0.0, 0.1, 40)].astype(F32), 1.0),
    }


@pytest.mark.parametrize("name", list(_clouds()))
def test_oracle_equals_a_literal_statement(name):
    pts, size = _clouds()[name]
    got = vfr.voxel_filter(pts, size)
    want = _py_voxel(pts, size)
    assert got.dtype == F32 and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    if name == "one_voxel":
        assert len(got) == 1
    if name == "own_voxel":
        assert np.array_equal(got, pts)
    if name == "single":
        assert np.array_equal(got, pts)
    if name == "negative_zero":
        assert len(got) == 1 and got[0, 0] == 0 and np.signbit(got[0, 0])


def test_oracle_keeps_first_points_in_input_order():
    # the grid starts at the minima (-0.5, 0.25): x voxels [-0.5, 0.5), [0.5, 1.5), [1.5, 2.5), one row.  Points 0 and
    # 4 share voxel 0, point 1 is alone in voxel 2, points 2 and 3 share voxel 1: the output follows the first points
    pts = np.array([[0.25, 0.25], [1.5, 0.5], [0.75, 0.75], [1.25, 0.25], [-0.5, 0.5]], F32)
    got = vfr.voxel_filter(pts, 1.0)
    want = np.array([[-0.125, 0.375], [1.5, 0.5], [1.0, 0.5]], F32)
    assert np.array_equal(got, want)


def test_oracle_reports_the_voxel_count_overflow():
    pts = np.array([[0, 0], [1000, 1000]], F32)
    with pytest.raises(vfr.VoxelOverflow):
        vfr.voxel_filter(pts, 0.01)  # 100 001^2 voxels
    assert len(vfr.voxel_filter(pts, 0.5)) == 2  # 2 001^2 fits
    with pytest.raises(vfr.VoxelOverflow):
        vfr.data_filters(pts, [(vfr.MAX_DIST, -1, 5000.0), (vfr.VOXEL, 1, 0.01)])
    # a distance filter before the voxel filter shrinks the grid it spans
    assert len(vfr.data_filters(pts, [(vfr.MAX_DIST, -1, 10.0), (vfr.VOXEL, 1, 0.01)])) == 1
    with pytest.raises(vfr.VoxelOverflow):
        vfr.icp(pts, pts, filters=vfr.IcpFilters(reference=[(vfr.VOXEL, 1, 0.01)]))


# ------------------------------------------------------------------------------------------ oracle: chains
CHAINS = [
    [(vfr.VOXEL, 1, 0.5)],
    [(vfr.MAX_DIST, -1, 12.0), (vfr.VOXEL, 1, 0.4)],
    [(vfr.VOXEL, 1, 0.3), (vfr.MIN_DIST, 0, -2.0)],
    [(vfr.OCTREE, 2, 0.2), (vfr.VOXEL, 1, 0.6)],
    [(vfr.VOXEL, 1, 0.25), (ofr.OCTREE, 3, 0.6), (vfr.MAX_DIST, 0, 5.0), (vfr.VOXEL, 1, 0.9)],
]


def _np_chain(pts, chain):
    """The chain as one step after the other: numpy masks for the distance filters, the literal voxel statement, and
    the octree oracle alone (tested against its own statement in test_icp_octree_filter_cpu.py)."""
    pts = np.asarray(pts, F32).reshape(-1, 2)
    for kind, dim, dist in chain:
        if kind == vfr.VOXEL:
            pts = _py_voxel(pts, dist)
        elif kind == vfr.OCTREE:
            pts = ofr.octree_filter(pts, dist, dim)
        else:
            pts = _np_data_filters(pts, [(kind, dim, dist)])
    return pts


@pytest.mark.parametrize("chain", range(len(CHAINS)))
def test_oracle_mixed_chains_equal_the_composition(chain):
    rng = np.random.default_rng(chain)
    pts = rng.uniform(-15, 15, (2000, 2)).astype(F32)
    pts[:300] = np.round(pts[:300] * 4) / 4  # on voxel boundaries
    got = vfr.data_filters(pts, CHAINS[chain])
    assert got.dtype == F32 and np.array_equal(got.view(np.uint32), _np_chain(pts, CHAINS[chain]).view(np.uint32))


@pytest.mark.parametrize("case", ["reading", "reference", "both", "trim_median"])
def test_oracle_one_iteration_is_the_computation_on_the_prefiltered_clouds(case):
    s, t, T = synth.make_icp_pair(21, n_source=1500, n_target=6000)
    rd = [(vfr.VOXEL, 1, 0.3), (vfr.MAX_DIST, -1, 20.0)] if case != "reference" else []
    rf = [(vfr.MIN_DIST, 0, -25.0), (vfr.VOXEL, 1, 0.2)] if case != "reading" else []
    kw = dict(median_factor=2.0) if case == "trim_median" else {}
    prm = orc.IcpParams(max_iterations=1, smooth_length=0)
    got = vfr.icp(s, t, T.astype(F32), prm, vfr.IcpFilters(reading=rd, reference=rf, **kw))
    s2, t2 = vfr.data_filters(s, rd), vfr.data_filters(t, rf)
    assert len(s2) < len(s) or len(t2) < len(t)
    st, inl, _ = _np_one_iteration(s2, t2, T.astype(F32), prm, vfr.IcpFilters(**kw))
    assert (got["status"], got["inliers"], got["iterations"]) == (st, inl, 1)
    same = vfr.icp(s2, t2, T.astype(F32), prm, vfr.IcpFilters(**kw))
    assert np.array_equal(got["T"], same["T"])
