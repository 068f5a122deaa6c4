"""CPU-only: OctreeGridDataPointsFilter in the ICP data-filter chains.

  * parse_icp_yaml reads the module in either chain: upstream's defaults, every accepted and rejected parameter, the
    fifth data filter of a cloud, and the module after the normals filter.
  * oracle/octree_filter_ref.c's octree filter: the medoid sampler is orc_downsample point for point (without the
    15-level cut where the cloud is deeper than that); the first-point and centroid samplers equal a literal recursive
    quadtree written here, on random, lattice-tie, collinear, coincident, single-point and deeper-than-15-level clouds.
  * oracle/octree_filter_ref.c's chains: those mixing distance and octree filters equal the numpy composition of the
    steps, and one iteration through an octree chain is the direct computation on the pre-filtered clouds.
"""
import numpy as np
import pytest

from oracle import octree_filter_ref as ofr
from oracle import oracle as orc
from sonar_slam_b200 import _lib, synth
from sonar_slam_b200.bruce_slam import pcl
from test_icp_filters_cpu import _np_data_filters, _np_one_iteration, _yaml

F32 = np.float32
OCT = "OctreeGridDataPointsFilter"
MAXD = "MaxDistDataPointsFilter: {dim: -1, maxDist: 25.0}"
NORMALS = "SurfaceNormalDataPointsFilter: {knn: 5}"


# ------------------------------------------------------------------------------------------ parser
def test_parser_reads_the_octree_filter_in_either_chain():
    # samplingMethod defaults to 0 (first point); maxPointByNode and buildParallel are ignored once a size is given
    p = pcl.parse_icp_yaml(_yaml(reading=[f"{OCT}: {{maxSizeByNode: 0.2}}"]))
    assert p.filters.data_filters("reading") == [(_lib.OCTREE, 0, pytest.approx(0.2))] and p.filters.n_reference == 0
    for method in (0, 2, 3):
        q = f"{OCT}: {{maxSizeByNode: 0.5, samplingMethod: {method}, maxPointByNode: 7, buildParallel: 0}}"
        p = pcl.parse_icp_yaml(_yaml(reference=[q]))
        assert p.filters.data_filters("reference") == [(_lib.OCTREE, method, 0.5)] and p.filters.n_reading == 0
    # mixed with the distance filters, in listed order, before the normals filter
    p = pcl.parse_icp_yaml(_yaml(reading=[MAXD, f"{OCT}: {{maxSizeByNode: 1, samplingMethod: 3}}"],
                                 reference=[f"{OCT}: {{maxSizeByNode: 0.25, samplingMethod: 2}}", MAXD, NORMALS],
                                 minimizer="PointToPlaneErrorMinimizer"))
    assert p.minimizer == 1
    assert p.filters.data_filters("reading") == [(_lib.MAX_DIST, -1, 25.0), (_lib.OCTREE, 3, 1.0)]
    assert p.filters.data_filters("reference") == [(_lib.OCTREE, 2, 0.25), (_lib.MAX_DIST, -1, 25.0)]
    # the same octree twice is a chain, not a duplicate; four per cloud
    p = pcl.parse_icp_yaml(_yaml(reading=[f"{OCT}: {{maxSizeByNode: 0.3}}"] * 2 + [MAXD]))
    assert p.filters.n_reading == 3


@pytest.mark.parametrize("bad", [
    f"{OCT}: {{maxSizeByNode: -0.5}}",
    f"{OCT}: {{maxSizeByNode: .nan}}",
    f"{OCT}: {{maxSizeByNode: .inf}}",
    f"{OCT}: {{maxSizeByNode: -.inf}}",
    f"{OCT}: {{maxSizeByNode: 0.5, samplingMethod: 4}}",
    f"{OCT}: {{maxSizeByNode: 0.5, samplingMethod: -1}}",
])
def test_parser_rejects_bad_octree_values(bad):
    for side in ("reading", "reference"):
        with pytest.raises(ValueError):
            pcl.parse_icp_yaml(_yaml(**{side: [bad]}))


@pytest.mark.parametrize("bad, why", [
    (f"{OCT}: {{maxSizeByNode: 0.5, samplingMethod: 1}}", "random"),
    (f"{OCT}", "maxPointByNode"),                                   # no size: the point-count criterion
    (f"{OCT}: {{maxPointByNode: 3}}", "maxPointByNode"),
    (f"{OCT}: {{maxSizeByNode: 0, samplingMethod: 3}}", "maxPointByNode"),
])
def test_parser_rejects_unimplemented_octree_settings(bad, why):
    for side in ("reading", "reference"):
        with pytest.raises(NotImplementedError, match=why):
            pcl.parse_icp_yaml(_yaml(**{side: [bad]}))


def test_parser_rejects_a_fifth_filter_and_an_octree_after_the_normals():
    oct_ = f"{OCT}: {{maxSizeByNode: 0.3}}"
    with pytest.raises(NotImplementedError, match="more than 4"):
        pcl.parse_icp_yaml(_yaml(reading=[oct_, MAXD, oct_, "MinDistDataPointsFilter: {minDist: 0.5}", oct_]))
    with pytest.raises(NotImplementedError, match="SurfaceNormalDataPointsFilter"):
        pcl.parse_icp_yaml(_yaml(reference=[NORMALS, oct_], minimizer="PointToPlaneErrorMinimizer"))
    assert pcl.parse_icp_yaml(_yaml(reference=[oct_, NORMALS], minimizer="PointToPlaneErrorMinimizer")).minimizer == 1


# ------------------------------------------------------------------------------------------ oracle: the tree
def _py_quadtree(pts, size, sampler, max_depth=15):
    """A second, literal statement of the octree filter, recursive over Python lists with numpy float32 scalars:
    bounding square, split while 2 * radius > size and more than one point and the node is above `max_depth`,
    children by (x > cx) | (y > cy) << 1 visited in index order; sampler 0 keeps the leaf's first member, 2 the
    float32 sequential means of x and y.  Shares no code with oracle/octree_filter_ref.c."""
    f = np.float32
    pts = np.asarray(pts, np.float32)
    if len(pts) == 0:
        return np.zeros((0, 2), np.float32)
    mn, mx = pts.min(0), pts.max(0)
    rad = mx - mn
    cx, cy = mn[0] + rad[0] * f(0.5), mn[1] + rad[1] * f(0.5)
    radius = (rad[0] if rad[0] >= rad[1] else rad[1]) * f(0.5)
    out = []

    def leaf(members):
        if sampler == 0:
            out.append(pts[members[0]])
            return
        sx, sy = f(0), f(0)
        for i in members:
            sx, sy = f(sx + pts[i, 0]), f(sy + pts[i, 1])
        out.append(np.array([sx / f(len(members)), sy / f(len(members))], np.float32))

    def build(members, cx, cy, radius, depth):
        if not members:
            return
        if float(radius) * 2.0 <= float(f(size)) or len(members) <= 1 or depth >= max_depth:
            leaf(members)
            return
        kids = [[], [], [], []]
        for i in members:
            kids[int(pts[i, 0] > cx) | (int(pts[i, 1] > cy) << 1)].append(i)
        hr = radius * f(0.5)
        for k in range(4):
            build(kids[k], cx + (hr if k & 1 else -hr), cy + (hr if k & 2 else -hr), hr, depth + 1)

    build(list(range(len(pts))), cx, cy, radius, 0)
    return np.array(out, np.float32).reshape(-1, 2)


def _clouds():
    rng = np.random.default_rng(11)
    lattice = (np.round(rng.uniform(-20, 20, (1500, 2)) / 0.25) * 0.25).astype(F32)  # ties on every split line
    t = rng.uniform(0, 1, 600).astype(F32)
    deep = np.concatenate([rng.uniform(0, 1e-5, (300, 2)), [[0.0, 0.0], [1000.0, 1000.0]]]).astype(F32)
    return {
        "random": (rng.uniform(-30, 30, (2500, 2)).astype(F32), 0.7),
        "sonar": (synth.make_icp_pair(3, n_source=800, n_target=4000)[1], 0.3),
        "lattice": (lattice, 0.5),
        "collinear": (np.c_[t * 40 - 20, t * 10].astype(F32), 0.4),
        "coincident": (np.repeat(np.array([[1.5, -2.25], [1.5, -2.25], [3.0, 4.0]], F32), 50, axis=0), 0.1),
        "single": (np.array([[7.0, -3.5]], F32), 0.2),
        "deep": (deep, 1e-9),  # 1000 m / 2^15 is still far above the size: the 15-level cut decides the leaves
    }


@pytest.mark.parametrize("name", list(_clouds()))
def test_oracle_medoid_is_downsample(name):
    pts, size = _clouds()[name]
    want, _ = orc.downsample(pts, size)
    got = ofr.octree_filter(pts, size, 3)
    if name == "deep":  # the uncut tree goes on splitting the 10-micron cluster
        assert len(want) > len(got)
        got = ofr.octree_filter(pts, size, 3, max_depth=None)
    assert got.dtype == F32 and np.array_equal(got, want)


@pytest.mark.parametrize("sampler", [0, 2])
@pytest.mark.parametrize("name", list(_clouds()))
def test_oracle_first_point_and_centroid_equal_a_literal_quadtree(name, sampler):
    pts, size = _clouds()[name]
    got = ofr.octree_filter(pts, size, sampler)
    want = _py_quadtree(pts, size, sampler)
    assert got.dtype == F32 and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    if name == "deep":
        assert len(got) < len(_py_quadtree(pts, size, sampler, max_depth=10 ** 6))
    if name == "coincident":
        assert len(got) == 2
    if name == "single":
        assert np.array_equal(got, pts)


# ------------------------------------------------------------------------------------------ oracle: chains
CHAINS = [
    [(ofr.OCTREE, 0, 0.5)],
    [(ofr.MAX_DIST, -1, 12.0), (ofr.OCTREE, 2, 0.4)],
    [(ofr.OCTREE, 3, 0.3), (ofr.MIN_DIST, 0, -2.0)],
    [(ofr.MIN_DIST, -1, 2.0), (ofr.OCTREE, 0, 0.2), (ofr.MAX_DIST, 1, 6.0), (ofr.OCTREE, 2, 0.8)],
    [(ofr.OCTREE, 2, 0.25), (ofr.OCTREE, 3, 0.6), (ofr.MAX_DIST, 0, 5.0), (ofr.MIN_DIST, 1, -8.0)],
]


def _np_chain(pts, chain):
    """The chain as one step after the other: numpy masks for the distance filters, the literal quadtree (or
    orc.downsample for the medoid) for the octree."""
    pts = np.asarray(pts, F32).reshape(-1, 2)
    for kind, dim, dist in chain:
        if kind != ofr.OCTREE:
            pts = _np_data_filters(pts, [(kind, dim, dist)])
        elif dim == 3:
            pts = orc.downsample(pts, dist)[0] if len(pts) else pts
        else:
            pts = _py_quadtree(pts, dist, dim)
    return pts


@pytest.mark.parametrize("chain", range(len(CHAINS)))
def test_oracle_mixed_chains_equal_the_composition(chain):
    rng = np.random.default_rng(chain)
    pts = rng.uniform(-15, 15, (2000, 2)).astype(F32)
    pts[:300] = np.round(pts[:300] * 4) / 4  # lattice ties
    got = ofr.data_filters(pts, CHAINS[chain])
    assert got.dtype == F32 and np.array_equal(got.view(np.uint32), _np_chain(pts, CHAINS[chain]).view(np.uint32))


@pytest.mark.parametrize("case", ["reading", "reference", "both", "trim_median"])
def test_oracle_one_iteration_is_the_computation_on_the_prefiltered_clouds(case):
    s, t, T = synth.make_icp_pair(21, n_source=1500, n_target=6000)
    rd = [(ofr.OCTREE, 2, 0.3), (ofr.MAX_DIST, -1, 20.0)] if case != "reference" else []
    rf = [(ofr.MIN_DIST, 0, -25.0), (ofr.OCTREE, 3, 0.2)] if case != "reading" else []
    kw = dict(median_factor=2.0) if case == "trim_median" else {}
    prm = orc.IcpParams(max_iterations=1, smooth_length=0)
    got = ofr.icp(s, t, T.astype(F32), prm, ofr.IcpFilters(reading=rd, reference=rf, **kw))
    s2, t2 = ofr.data_filters(s, rd), ofr.data_filters(t, rf)
    assert len(s2) < len(s) or len(t2) < len(t)
    st, inl, _ = _np_one_iteration(s2, t2, T.astype(F32), prm, ofr.IcpFilters(**kw))
    assert (got["status"], got["inliers"], got["iterations"]) == (st, inl, 1)
    same = ofr.icp(s2, t2, T.astype(F32), prm, ofr.IcpFilters(**kw))
    assert np.array_equal(got["T"], same["T"])
