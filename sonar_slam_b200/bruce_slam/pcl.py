"""`bruce_slam.pcl` -- same names as the pybind11 module built from
bruce_slam/src/bruce_slam/cpp/pcl.cpp:176-214, running on the GPU through libsonarfe.

    remove_outlier(points[N,2|3], radius, min_points)          -> float32[M,2|3]      (pcl.cpp:54)
    downsample(points[N,2|3], resolution)                       -> float32[M,2|3]      (pcl.cpp:128)
    downsample(points[N,2|3], desc[N,d], resolution)            -> (points, desc)      (pcl.cpp:143)
    match(ref[N_t,2|3], in[N_s,2|3], knn, max_dist)             -> (int32[knn,N_s], float32[knn,N_s])  (:161)
    match_knn(ref[N_t,2|3], in[N_s,2|3], knn, max_dist)         -> the same for knn 1 .. 16 (match serves knn = 1)
    ICP().loadFromYaml(path) / .compute(source, target, guess)  -> (message, float32[3,3])   (:185-212)
        (the YAML's distance, octree and voxel-grid data filters and MinDist / MedianDist outlier filters included:
        parse_icp_yaml)
    ICP().compute(source[N,3], target[M,3], guess 4x4)          -> (message, float32[4,4])   (3-D, point-to-point)

Like pybind11 (`const PM::Matrix &` = Eigen float matrix) every array argument is converted to
float32; results are fresh float32 arrays.  Three columns are x, y, z, as fromEigen (pcl.cpp:18-50) reads them:
downsample then builds libpointmatcher's octree instead of the quadtree, match measures 3-D distances, and the
reference and query of a match must have the same number of columns.  ICP registers 3-column clouds with 4x4 guesses
through libpointmatcher's 3-D point-to-point chain (the 3-D scan matcher takes no point-to-plane minimiser and no ICP
filters: a YAML selecting them raises NotImplementedError on 3-column input).  Not provided: density_filter (dead code in the
reference: its only call site is commented out, feature_extraction.py:246) and
ICP.getCovariance (never called from Python) -- both raise NotImplementedError.
"""
import math
import os

import numpy as np

from .. import _lib


def _points(a, name, cols=(2, 3)):
    a = np.asarray(a)
    if a.ndim != 2 or a.dtype.kind not in "buif" or (a.shape[1] not in cols and a.shape[0] != 0):
        raise TypeError(f"pcl: incompatible function arguments ({name} must be a real [N,{'|'.join(map(str, cols))}] array)")
    return np.ascontiguousarray(a, dtype=np.float32)


def remove_outlier(mat_in, radius, min_points):
    """Points with at least min_points others within radius, in input order.  Any size, whole maps included."""
    pts = _points(mat_in, "points")
    n, dim = pts.shape
    if n == 0:
        return pts.copy()
    ctx = _lib.default_context()
    out = np.empty_like(pts)
    idx = np.empty(n, np.int32)
    m = np.zeros(1, np.int32)
    _lib.check(ctx.lib.sfe_remove_outlier_host(ctx.handle, _lib.ptr(pts), n, dim, float(radius), int(min_points),
                                               _lib.ptr(out), _lib.ptr(idx), _lib.ptr(m)), "remove_outlier")
    return out[:int(m[0])].copy()


def downsample(mat_in, *args):
    """downsample(points, resolution) or downsample(points, desc, resolution)."""
    if len(args) == 1:
        desc, resolution = None, args[0]
    elif len(args) == 2:
        desc, resolution = args
    else:
        raise TypeError("pcl.downsample: incompatible function arguments")
    pts = _points(mat_in, "points")
    if desc is not None:
        desc = np.asarray(desc)
        if desc.ndim != 2 or len(desc) != len(pts):
            raise TypeError("pcl.downsample: descriptors must be [N,d]")
        desc = np.ascontiguousarray(desc, dtype=np.float32)
    n = len(pts)
    if n == 0:  # pcl.cpp:130,145: empty input comes straight back
        return pts.copy() if desc is None else (pts.copy(), desc.copy())
    ctx = _lib.default_context()
    out = np.empty_like(pts)
    idx = np.empty(n, np.int32)
    m = np.zeros(1, np.int32)
    _lib.check(ctx.lib.sfe_downsample_host(ctx.handle, _lib.ptr(pts), n, pts.shape[1], float(resolution), _lib.ptr(out),
                                           _lib.ptr(idx), _lib.ptr(m)), "downsample")
    k = int(m[0])
    if desc is None:
        return out[:k].copy()
    return out[:k].copy(), desc[idx[:k]].copy()


def density_filter(*args, **kwargs):
    raise NotImplementedError("pcl.density_filter is dead code in the reference (its only call site is commented "
                              "out, feature_extraction.py:246) and is not provided")


def _match_clouds(mat_ref, mat_in):
    """ref and in as float32 [N,2] or [N,3] arrays with the same number of columns (libnabo rejects a query whose
    dimension differs from the tree's)."""
    ref = _points(mat_ref, "ref")
    pts = _points(mat_in, "in")
    if ref.shape[1] != pts.shape[1]:
        raise TypeError(f"pcl: incompatible function arguments (ref has {ref.shape[1]} columns, in has "
                        f"{pts.shape[1]})")
    return ref, pts


def match(mat_ref, mat_in, knn, max_dist):
    """libnabo KD-tree match, knn = 1: (ids [1,N] int32, squared dists [1,N] float32).  References of any size (whole
    maps run as a grid in global memory, with the same results).  [N,3] clouds: 3-D distances."""
    if int(knn) != 1:
        raise NotImplementedError("pcl.match: only knn = 1 is implemented (the only value the reference uses, "
                                  "slam.py:418)")
    ref, pts = _match_clouds(mat_ref, mat_in)
    ids = np.empty((1, len(pts)), np.int32)
    dists = np.empty((1, len(pts)), np.float32)
    if len(pts):
        ctx = _lib.default_context()
        if pts.shape[1] == 3:
            _lib.check(ctx.lib.sfe_match_dim_host(ctx.handle, _lib.ptr(ref), len(ref), _lib.ptr(pts), len(pts), 3,
                                                  float(max_dist), _lib.ptr(ids), _lib.ptr(dists)), "match")
        else:
            _lib.check(ctx.lib.sfe_match_host(ctx.handle, _lib.ptr(ref), len(ref), _lib.ptr(pts), len(pts),
                                              float(max_dist), _lib.ptr(ids), _lib.ptr(dists)), "match")
    return ids, dists


KNN_MAX = 16  # the largest knn match_knn serves (GRID_KNN_MAX, csrc/grid.cuh)


def match_knn(mat_ref, mat_in, knn, max_dist):
    """libnabo KD-tree match for any knn up to 16 (what pcl.cpp:161-174 computes for knn > 1): for every query point
    its knn nearest reference points within max_dist, nearest first (ties: lower reference index), as (ids [knn,N]
    int32, squared dists [knn,N] float32); slots with no neighbour left hold -1 / +inf.  Row 0 is match(..., 1, ...)'s
    result.  References of any size (whole maps run as a grid in global memory, with the same results).  [N,3] clouds:
    3-D distances."""
    knn = int(knn)
    if knn < 1:
        raise ValueError(f"pcl.match_knn: knn must be at least 1 (got {knn})")
    if knn > KNN_MAX:
        raise NotImplementedError(f"pcl.match_knn: knn {knn} is not supported (at most {KNN_MAX})")
    ref, pts = _match_clouds(mat_ref, mat_in)
    ids = np.empty((knn, len(pts)), np.int32)
    dists = np.empty((knn, len(pts)), np.float32)
    if len(pts):
        ctx = _lib.default_context()
        if pts.shape[1] == 3:
            _lib.check(ctx.lib.sfe_match_knn_dim_host(ctx.handle, _lib.ptr(ref), len(ref), _lib.ptr(pts), len(pts), 3,
                                                      knn, float(max_dist), _lib.ptr(ids), _lib.ptr(dists)),
                       "match_knn")
        else:
            _lib.check(ctx.lib.sfe_match_knn_host(ctx.handle, _lib.ptr(ref), len(ref), _lib.ptr(pts), len(pts), knn,
                                                  float(max_dist), _lib.ptr(ids), _lib.ptr(dists)), "match_knn")
    return ids, dists


# ------------------------------------------------------------------------------------------ ICP
_SUPPORTED = ("the modules of the shipped bruce_slam/config/icp.yaml are implemented, plus its commented-out "
              "PointToPlaneErrorMinimizer with a SurfaceNormalDataPointsFilter on the reference, the Max/MinDist data "
              "filters, the OctreeGridDataPointsFilter with maxSizeByNode and samplingMethod 0, 2 or 3, the "
              "VoxelGridDataPointsFilter with vSizeX == vSizeY and useCentroid 1, the "
              "SamplingSurfaceNormalDataPointsFilter as the last reference filter (knn 3..64, samplingMethod 1, or 0 "
              "with ratio 1), a SurfaceNormalDataPointsFilter on the reading (knn 3..16) followed by distance filters "
              "and ShadowDataPointsFilter, the MinDist / MedianDist "
              "outlier filters and one RobustOutlierFilter with scaleEstimator none or fixed")
_DATA_FILTERS = {"MaxDistDataPointsFilter": ("maxDist", _lib.MAX_DIST), "MinDistDataPointsFilter": ("minDist", _lib.MIN_DIST)}


def _data_filter(name, p):
    """MaxDist / MinDistDataPointsFilter {dim, maxDist | minDist} -> (kind, dim, dist); upstream defaults dim -1, 1 m."""
    key, kind = _DATA_FILTERS[name]
    dim, dist = int(p.get("dim", -1)), float(p.get(key, 1.0))
    if dim not in (-1, 0, 1):  # libpointmatcher: InvalidParameter for a dimension the 2-D cloud does not have
        raise ValueError(f"ICP yaml: {name} dim {dim} (2-D clouds: -1, 0 or 1)")
    if math.isnan(dist):
        raise ValueError(f"ICP yaml: {name} {key} is NaN")
    return kind, dim, dist


_OCTREE = "OctreeGridDataPointsFilter"


def _octree_filter(p):
    """OctreeGridDataPointsFilter {maxSizeByNode, samplingMethod, maxPointByNode, buildParallel} -> (OCTREE, sampling
    method, maxSizeByNode): the quadtree of pcl.downsample with one point per leaf -- 0 the first (lowest-index) member,
    upstream's default; 2 the float32 centroid; 3 the medoid.  maxPointByNode (moot once a size is given) and
    buildParallel (results do not depend on it) are ignored."""
    size = float(p.get("maxSizeByNode", 0.0))
    if not math.isfinite(size) or size < 0:
        raise ValueError(f"ICP yaml: {_OCTREE} maxSizeByNode {size} must be finite and non-negative")
    if size == 0:
        # coincident points make libpointmatcher's point-count recursion depend on float underflow, which the
        # device's 15-level tree cannot follow
        raise NotImplementedError(f"ICP yaml: {_OCTREE} without maxSizeByNode (the maxPointByNode criterion) is not "
                                  "implemented: give maxSizeByNode > 0")
    method = p.get("samplingMethod", 0)
    if method not in (0, 1, 2, 3) or isinstance(method, bool):
        raise ValueError(f"ICP yaml: {_OCTREE} samplingMethod {method!r} (0 first point, 1 random, 2 centroid, "
                         "3 medoid)")
    if method == 1:
        raise NotImplementedError(f"ICP yaml: {_OCTREE} samplingMethod 1 (random sampling) is not implemented: its "
                                  "result depends on a random generator (0, 2 and 3 are)")
    return _lib.OCTREE, int(method), size


_VOXEL = "VoxelGridDataPointsFilter"


def _voxel_filter(p):
    """VoxelGridDataPointsFilter {vSizeX, vSizeY, vSizeZ, useCentroid, averageExistingDescriptors} -> (VOXEL, 1, vSize):
    the first point of every voxel, in point order, holding its voxel's float32 centroid.  vSizeZ is moot on 2-D clouds
    and averageExistingDescriptors on clouds without descriptors; both are ignored."""
    sx, sy = float(p.get("vSizeX", 1.0)), float(p.get("vSizeY", 1.0))
    for axis, v in (("vSizeX", sx), ("vSizeY", sy)):
        if not math.isfinite(v) or v <= 0:
            raise ValueError(f"ICP yaml: {_VOXEL} {axis} {v} must be finite and positive")
    if sx != sy:
        raise NotImplementedError(f"ICP yaml: {_VOXEL} with vSizeX {sx} != vSizeY {sy} is not implemented: give one "
                                  "size for both axes")
    centroid = p.get("useCentroid", 1)
    if centroid not in (0, 1):
        raise ValueError(f"ICP yaml: {_VOXEL} useCentroid {centroid!r} (0 or 1)")
    if not centroid:
        raise NotImplementedError(f"ICP yaml: {_VOXEL} useCentroid 0 (the voxel centre) is not implemented: its "
                                  "formula cannot be checked against upstream (1, the centroid, is)")
    return _lib.VOXEL, 1, sx


_SAMPLING = "SamplingSurfaceNormalDataPointsFilter"
SAMPLING_KNN_MAX = 64  # the largest box the device's sampling-normals stage takes


def _sampling_filter(p):
    """SamplingSurfaceNormalDataPointsFilter {knn, samplingMethod, ratio, maxBoxDim, keepNormals, ...} -> (knn,
    (SAMPLING_NORMALS, samplingMethod, maxBoxDim), keepNormals).  Upstream defaults knn 7, samplingMethod 0, ratio 0.5,
    maxBoxDim inf, keepNormals 1.  averageExistingDescriptors, keepDensities, keepEigenValues and keepEigenVectors have
    no consumer here and are ignored."""
    knn = p.get("knn", 7)
    if isinstance(knn, bool) or int(knn) != knn or not 3 <= int(knn) <= SAMPLING_KNN_MAX:
        raise NotImplementedError(f"ICP yaml: {_SAMPLING} knn {knn!r} (an integer, 3..{SAMPLING_KNN_MAX})")
    method = p.get("samplingMethod", 0)
    if method not in (0, 1) or isinstance(method, bool):
        raise ValueError(f"ICP yaml: {_SAMPLING} samplingMethod {method!r} (0 random, 1 centroid)")
    ratio = float(p.get("ratio", 0.5))
    if not 0.0 < ratio <= 1.0:
        raise ValueError(f"ICP yaml: {_SAMPLING} ratio {ratio} must lie in (0, 1]")
    if method == 0 and ratio != 1.0:
        raise NotImplementedError(f"ICP yaml: {_SAMPLING} samplingMethod 0 with ratio {ratio} (random sampling) is not "
                                  "implemented: its result depends on a random generator (1, and 0 with ratio 1, are)")
    box = float(p.get("maxBoxDim", float("inf")))
    if math.isnan(box) or box < 0:
        raise ValueError(f"ICP yaml: {_SAMPLING} maxBoxDim {box} must be non-negative")
    return int(knn), (_lib.SAMPLING_NORMALS, int(method), box), bool(int(p.get("keepNormals", 1)))


_NORMALS = "SurfaceNormalDataPointsFilter"
_SHADOW = "ShadowDataPointsFilter"


def _reading_normals_filter(p):
    """SurfaceNormalDataPointsFilter {knn, epsilon, keepNormals, ...} on the reading -> (NORMALS, knn, 0.0), or None
    with keepNormals 0 (nothing reads the normals then).  Upstream defaults knn 5, epsilon 0, keepNormals 1;
    keepDensities, keepEigenValues, keepEigenVectors and keepMatchedIds have no consumer here and are ignored."""
    knn = p.get("knn", 5)
    if isinstance(knn, bool) or int(knn) != knn or not 3 <= int(knn) <= 16:
        raise NotImplementedError(f"ICP yaml: reading {_NORMALS} knn {knn!r} (an integer, 3..16)")
    if float(p.get("epsilon", 0)) != 0:
        raise NotImplementedError(f"ICP yaml: reading {_NORMALS} epsilon {p['epsilon']} (approximate neighbours; 0 is "
                                  "implemented)")
    return (_lib.NORMALS, int(knn), 0.0) if int(p.get("keepNormals", 1)) else None


def _shadow_filter(p):
    """ShadowDataPointsFilter {eps} -> (SHADOW, 0, eps); upstream default 0.1 rad."""
    eps = float(p.get("eps", 0.1))
    if not math.isfinite(eps):
        raise ValueError(f"ICP yaml: {_SHADOW} eps {eps} must be finite")
    return _lib.SHADOW, 0, eps


_RESAMPLERS = {_OCTREE: _octree_filter, _VOXEL: _voxel_filter}
_ROBUST = "RobustOutlierFilter"


def _robust_filter(p):
    """RobustOutlierFilter {robustFct, tuning, approximation, scaleEstimator, nbIterationForScale, distanceType} ->
    _lib.IcpRobust.  Upstream defaults robustFct cauchy, tuning 1, approximation inf, distanceType point2point.  With
    scaleEstimator none or fixed the scale is 1 and the tuning is k itself; nbIterationForScale is then moot."""
    fct = str(p.get("robustFct", "cauchy"))
    if fct == "student":
        raise NotImplementedError(f"ICP yaml: {_ROBUST} robustFct student is not implemented ({_SUPPORTED})")
    if fct not in _lib.ROBUST_FCT:
        raise ValueError(f"ICP yaml: {_ROBUST} robustFct {fct!r} ({', '.join(_lib.ROBUST_FCT)})")
    if "scaleEstimator" not in p:
        raise NotImplementedError(f"ICP yaml: {_ROBUST} without scaleEstimator is not implemented: the default "
                                  "estimator cannot be checked against upstream; give scaleEstimator none or fixed")
    scale = str(p["scaleEstimator"])
    if scale in ("mad", "berg"):
        raise NotImplementedError(f"ICP yaml: {_ROBUST} scaleEstimator {scale} is not implemented (none and fixed are)")
    if scale not in ("none", "fixed"):
        raise ValueError(f"ICP yaml: {_ROBUST} scaleEstimator {scale!r} (mad, berg, none or fixed)")
    dist = str(p.get("distanceType", "point2point"))
    if dist == "point2plane":
        raise NotImplementedError(f"ICP yaml: {_ROBUST} distanceType point2plane is not implemented (point2point is)")
    if dist != "point2point":
        raise ValueError(f"ICP yaml: {_ROBUST} distanceType {dist!r} (point2point or point2plane)")
    k = float(p.get("tuning", 1.0))
    if not math.isfinite(k) or k <= 0:
        raise ValueError(f"ICP yaml: {_ROBUST} tuning {k} must be finite and positive")
    approx = float(p.get("approximation", float("inf")))
    if math.isnan(approx):
        raise ValueError(f"ICP yaml: {_ROBUST} approximation is NaN")
    return _lib.IcpRobust(fct, k, approx)


def parse_icp_yaml(text):
    """libpointmatcher ICP YAML (the subset described by _SUPPORTED) -> _lib.IcpConfig: the IcpParams the shipped modules
    set, with `.filters` = the _lib.IcpFilters of the distance, octree and voxel-grid data filters, in their listed
    order, and the MinDist / MedianDist outlier filters (None when the YAML has none of them), and `.robust` = the
    _lib.IcpRobust of its RobustOutlierFilter (None without one)."""
    import yaml
    cfg = yaml.safe_load(text) or {}

    def one(node):  # "Name" | {"Name": {params}} -> (name, params)
        if isinstance(node, str):
            return node, {}
        if isinstance(node, dict) and len(node) == 1:
            (name, prm), = node.items()
            return name, (prm or {})
        raise ValueError(f"ICP yaml: cannot parse module {node!r}")

    def add_data_filter(chain, name, p, which):
        f = _RESAMPLERS[name](p) if name in _RESAMPLERS else _data_filter(name, p)
        if name not in _RESAMPLERS and (name,) + f in chain:
            raise ValueError(f"ICP yaml: {name} {p} appears twice in {which}DataPointsFilters")
        if len(chain) == _lib.MAX_DATA_FILTERS:
            raise NotImplementedError(f"ICP yaml: more than {_lib.MAX_DATA_FILTERS} {which}DataPointsFilters")
        chain.append((name,) + f)

    prm = _lib.IcpConfig(outlier_max_dist=-1.0, trim_ratio=-1.0, max_iterations=40, smooth_length=0)
    reading, reference, outlier, robust = [], [], {}, None
    reading_normals = False  # a reading SurfaceNormalDataPointsFilter that keeps its normals came before
    for node in cfg.get("readingDataPointsFilters") or []:
        name, p = one(node)
        if name == _NORMALS:
            if reading_normals:
                raise NotImplementedError(f"ICP yaml: a second reading {_NORMALS} ({_SUPPORTED})")
            f = _reading_normals_filter(p)
            if f:  # (keepNormals 0: a no-op)
                if len(reading) == _lib.MAX_DATA_FILTERS:
                    raise NotImplementedError(f"ICP yaml: more than {_lib.MAX_DATA_FILTERS} readingDataPointsFilters")
                reading.append((name,) + f)
                reading_normals = True
            continue
        if name == _SHADOW:
            if not reading_normals:
                # libpointmatcher: InvalidField when the cloud carries no normals descriptor
                raise ValueError(f"ICP yaml: {_SHADOW} needs the reading's normals (InvalidField: no descriptor "
                                 f"normals): put a {_NORMALS} with keepNormals 1 before it in readingDataPointsFilters")
            f = _shadow_filter(p)
            if len(reading) == _lib.MAX_DATA_FILTERS:
                raise NotImplementedError(f"ICP yaml: more than {_lib.MAX_DATA_FILTERS} readingDataPointsFilters")
            reading.append((name,) + f)
            continue
        if name not in _DATA_FILTERS and name not in _RESAMPLERS:
            raise NotImplementedError(f"ICP yaml: reading filter {name} ({_SUPPORTED})")
        if name in _RESAMPLERS and reading_normals:  # the normals would need down-sampling with the points
            raise NotImplementedError(f"ICP yaml: reading filter {name} after {_NORMALS} ({_SUPPORTED}: only the "
                                      f"distance filters and {_SHADOW} may follow it)")
        add_data_filter(reading, name, p, "reading")
    have_normals, normal_source = False, None
    for node in cfg.get("referenceDataPointsFilters") or []:
        name, p = one(node)
        if name == _SHADOW:
            raise NotImplementedError(f"ICP yaml: reference filter {_SHADOW} ({_SUPPORTED}: on the reading only)")
        if name in _DATA_FILTERS or name in _RESAMPLERS:
            if normal_source:  # the normals would describe points the filter then removes
                raise NotImplementedError(f"ICP yaml: {name} after {normal_source} ({_SUPPORTED}: the data filters go "
                                          "before it)")
            add_data_filter(reference, name, p, "reference")
            continue
        if name in (_SAMPLING, "SurfaceNormalDataPointsFilter") and normal_source:
            raise NotImplementedError(f"ICP yaml: {name} after {normal_source}: one source of normals per reference "
                                      f"cloud ({_SUPPORTED})")
        if name == _SAMPLING:
            knn, f, keep = _sampling_filter(p)
            if len(reference) == _lib.MAX_DATA_FILTERS:
                raise NotImplementedError(f"ICP yaml: more than {_lib.MAX_DATA_FILTERS} referenceDataPointsFilters")
            reference.append((name,) + f)
            prm.normals_knn, have_normals, normal_source = knn, keep, name
            continue
        # the one other reference filter: point-to-plane needs it, it attaches the "normals" descriptor
        if name != "SurfaceNormalDataPointsFilter" or float(p.get("epsilon", 0)) != 0:
            raise NotImplementedError(f"ICP yaml: reference filter {name} {p} ({_SUPPORTED})")
        if not int(p.get("keepNormals", 1)):
            continue
        prm.normals_knn = int(p.get("knn", 5))
        if not 3 <= prm.normals_knn <= 16:
            raise NotImplementedError(f"ICP yaml: SurfaceNormalDataPointsFilter knn {prm.normals_knn} (3..16)")
        have_normals, normal_source = True, name
    name, p = one(cfg.get("matcher", "KDTreeMatcher"))
    if name != "KDTreeMatcher" or int(p.get("knn", 1)) != 1 or float(p.get("epsilon", 0)) != 0:
        raise NotImplementedError(f"ICP yaml: matcher {name} {p} ({_SUPPORTED})")
    prm.matcher_max_dist = float(p.get("maxDist", float("inf")))
    for node in cfg.get("outlierFilters") or []:
        name, p = one(node)
        if name == "MaxDistOutlierFilter":
            prm.outlier_max_dist = float(p.get("maxDist", 1.0))
        elif name == "TrimmedDistOutlierFilter":
            prm.trim_ratio = float(p.get("ratio", 0.85))
        elif name in ("MinDistOutlierFilter", "MedianDistOutlierFilter"):
            if name in outlier:
                raise ValueError(f"ICP yaml: {name} appears twice in outlierFilters")
            # upstream defaults: minDist 1, factor 3
            v = float(p.get("minDist", 1.0)) if name == "MinDistOutlierFilter" else float(p.get("factor", 3.0))
            if not math.isfinite(v) or v < 0:
                raise ValueError(f"ICP yaml: {name} {p} needs a finite, non-negative value")
            outlier[name] = v
        elif name == _ROBUST:
            if robust is not None:
                raise NotImplementedError(f"ICP yaml: a second {_ROBUST} is not implemented ({_SUPPORTED})")
            robust = _robust_filter(p)
        else:
            raise NotImplementedError(f"ICP yaml: outlier filter {name} ({_SUPPORTED})")
    name, p = one(cfg.get("errorMinimizer", "PointToPointErrorMinimizer"))
    if name == "PointToPlaneErrorMinimizer":  # icp.yaml:18-19 (commented out upstream); 2-D clouds: force2D is moot
        if not have_normals:
            # libpointmatcher: DataPoints::getDescriptorViewByName throws InvalidField at the first iteration
            raise ValueError("ICP yaml: PointToPlaneErrorMinimizer needs the reference's normals "
                             "(InvalidField: Cannot find descriptor normals): add a SurfaceNormalDataPointsFilter "
                             "to referenceDataPointsFilters")
        prm.minimizer = 1
    elif name != "PointToPointErrorMinimizer":
        raise NotImplementedError(f"ICP yaml: error minimizer {name} ({_SUPPORTED})")
    prm.max_iterations = 40
    for node in cfg.get("transformationCheckers") or []:
        name, p = one(node)
        if name == "CounterTransformationChecker":
            prm.max_iterations = int(p.get("maxIterationCount", 40))
        elif name == "DifferentialTransformationChecker":
            prm.min_diff_rot = float(p.get("minDiffRotErr", 0.001))
            prm.min_diff_trans = float(p.get("minDiffTransErr", 0.001))
            prm.smooth_length = int(p.get("smoothLength", 3))
        else:
            raise NotImplementedError(f"ICP yaml: transformation checker {name} ({_SUPPORTED})")
    for f in ("matcher_max_dist", "outlier_max_dist", "trim_ratio", "min_diff_rot", "min_diff_trans"):
        if math.isnan(getattr(prm, f)):
            raise ValueError(f"ICP yaml: {f} is NaN")
    if prm.trim_ratio > 1.0:  # the quantile element floor(n * ratio) would lie past the sorted distances
        raise ValueError(f"ICP yaml: TrimmedDistOutlierFilter ratio {prm.trim_ratio} is above 1")
    if reading or reference or outlier:
        prm.filters = _lib.IcpFilters(min_dist=outlier.get("MinDistOutlierFilter", -1.0),
                                      median_factor=outlier.get("MedianDistOutlierFilter", -1.0),
                                      reading=[f[1:] for f in reading], reference=[f[1:] for f in reference])
    prm.robust = robust
    return prm


class ICP(object):
    """libpointmatcher PM::ICP as exposed by pcl.cpp:185-213.  Sources and targets of any size (map-to-map alignment
    included): the device picks the launch class from the clouds' sizes, and every class gives the same results."""

    def __init__(self):
        self.params = None  # no modules until loadFromYaml, like a default-constructed PM::ICP

    def loadFromYaml(self, filename):
        if not os.path.isfile(filename):
            # pcl.cpp:190-194 falls back to libpointmatcher's setDefault() (point-to-plane with sampled
            # surface normals), which is not implemented; the shipped icp.yaml values are used instead.
            print("Failed to load " + str(filename) + ". Use default configuration.")
            self.params = _lib.IcpParams()
            return
        with open(filename) as f:
            self.params = parse_icp_yaml(f.read())

    def compute(self, source, target, guess):
        res = self.compute_batch(source, target, [guess])
        return res["messages"][0], res["T"][0]

    def _dim(self, srcs, tgts):
        """The clouds' column count (2 or 3), after the checks the reference's module and the 3-D chain make: source
        and target with the same number of columns (TypeError), and for 3 columns a configuration the 3-D scan matcher
        runs (NotImplementedError, before any device call)."""
        if self.params is None:
            raise RuntimeError("You must setup a matcher before running ICP")
        dims = {c.shape[1] for c in list(srcs) + list(tgts) if c.shape[1] in (2, 3)}  # (empty [0,k] arrays pass _points)
        if len(dims) > 1:
            raise TypeError(f"pcl: incompatible function arguments (ICP clouds have {sorted(dims)} columns; source and "
                            "target must have the same number)")
        dim = dims.pop() if dims else 2
        if dim == 3:
            if self.params.minimizer != 0:
                raise NotImplementedError("ICP on 3-column clouds: PointToPlaneErrorMinimizer is not implemented in 3-D "
                                          "(3-D normals and the 6x6 system); use PointToPointErrorMinimizer")
            if self.params.flags & 2:
                raise NotImplementedError("ICP on 3-column clouds: float64 accumulation (flags bit 1) is not implemented")
            if _lib.icp_filters_of(self.params) is not None:
                raise NotImplementedError("ICP on 3-column clouds: data filters and MinDist / MedianDist outlier filters "
                                          "are not implemented in 3-D")
            if _lib.icp_robust_of(self.params) is not None:
                raise NotImplementedError("ICP on 3-column clouds: the RobustOutlierFilter is not implemented in 3-D")
        return dim

    @staticmethod
    def _guesses(guesses, dim):
        g = np.asarray(guesses, dtype=np.float32)
        if dim == 3 and (g.ndim < 2 or g.shape[-2:] != (4, 4)):
            raise ValueError(f"ICP on 3-column clouds takes 4x4 guesses (got shape {list(g.shape)})")
        return np.ascontiguousarray(g.reshape(-1, dim + 1, dim + 1))

    @staticmethod
    def _results(ctx, st):
        msgs = [ctx.lib.sfe_icp_status_message(int(s)).decode() for s in st]
        for s, m in zip(st, msgs):
            if int(s) in (5, 6):  # not ConvergenceErrors in libpointmatcher: they propagate as exceptions
                raise RuntimeError(m)
        return msgs

    def compute_batch(self, source, target, guesses):
        """All `guesses` (iterable of 3x3, or 4x4 for 3-column clouds) on the same cloud pair in one launch (N1: the
        loop of SLAM.compute_icp_with_cov, slam.py:346-358).  Returns dict(messages, T[n,3,3] (or [n,4,4]),
        iterations, inliers, status).  The target may be of any size (a whole map): above one CTA's shared memory it is
        sorted once into a grid in global memory that every guess reads, with the same results.  So may the source:
        above ops.icp_source_limit (about 8 400 points in 2-D, 11 000 in 3-D on an H100) its per-point arrays live in
        global memory (the global-source class), again with the same results."""
        if self.params is None:
            raise RuntimeError("You must setup a matcher before running ICP")
        src = _points(source, "source")
        tgt = _points(target, "target")
        dim = self._dim([src], [tgt])
        g = self._guesses(guesses, dim)
        n = len(g)
        T = np.empty((n, dim + 1, dim + 1), np.float32)
        iters, inl, st = (np.zeros(n, np.int32) for _ in range(3))
        ctx = _lib.default_context()
        import ctypes
        _lib.set_icp_filters(ctx, _lib.icp_filters_of(self.params))
        _lib.set_icp_robust(ctx, _lib.icp_robust_of(self.params))
        if dim == 3:
            _lib.check(ctx.lib.sfe_icp_dim_host(ctx.handle, ctypes.byref(self.params), _lib.ptr(src), len(src),
                                                _lib.ptr(tgt), len(tgt), 3, _lib.ptr(g), n, _lib.ptr(T),
                                                _lib.ptr(iters), _lib.ptr(inl), _lib.ptr(st)), "ICP.compute")
        else:
            _lib.check(ctx.lib.sfe_icp_host(ctx.handle, ctypes.byref(self.params), _lib.ptr(src), len(src),
                                            _lib.ptr(tgt), len(tgt), _lib.ptr(g), n, _lib.ptr(T), _lib.ptr(iters),
                                            _lib.ptr(inl), _lib.ptr(st)), "ICP.compute")
        msgs = self._results(ctx, st)
        return dict(messages=msgs, T=T, iterations=iters, inliers=inl, status=st)

    def compute_pairs(self, sources, targets, guesses):
        """Many cloud pairs, each with its own guesses, in ONE launch (sfe_icp_batch_host, or sfe_icp_batch_dim_host
        for 3-column clouds): pair k aligns sources[k] to targets[k] from every 3x3 (4x4) in guesses[k].  Returns a
        list with compute_batch's dict for every pair."""
        if self.params is None:
            raise RuntimeError("You must setup a matcher before running ICP")
        srcs = [_points(s, "source") for s in sources]
        tgts = [_points(t, "target") for t in targets]
        if not (len(srcs) == len(tgts) == len(guesses)):
            raise ValueError("sources, targets and guesses must have one entry per pair")
        dim = self._dim(srcs, tgts)
        gs = [self._guesses(g, dim) for g in guesses]
        counts = np.array([len(g) for g in gs], np.int64)
        n = int(counts.sum())
        if n == 0:
            return [dict(messages=[], T=np.empty((0, dim + 1, dim + 1), np.float32), iterations=np.zeros(0, np.int32),
                         inliers=np.zeros(0, np.int32), status=np.zeros(0, np.int32)) for _ in gs]

        def packed(clouds):
            off = np.zeros(len(clouds) + 1, np.int32)
            off[1:] = np.cumsum([len(c) for c in clouds])
            return np.ascontiguousarray(np.concatenate(clouds + [np.zeros((0, dim), np.float32)]), np.float32), off

        src, soff = packed(srcs)
        tgt, toff = packed(tgts)
        ids = np.ascontiguousarray(np.repeat(np.arange(len(gs), dtype=np.int32), counts))
        g = np.ascontiguousarray(np.concatenate(gs))
        T = np.empty((n, dim + 1, dim + 1), np.float32)
        iters, inl, st = (np.zeros(n, np.int32) for _ in range(3))
        ctx = _lib.default_context()
        import ctypes
        _lib.set_icp_filters(ctx, _lib.icp_filters_of(self.params))
        _lib.set_icp_robust(ctx, _lib.icp_robust_of(self.params))
        if dim == 3:
            _lib.check(ctx.lib.sfe_icp_batch_dim_host(ctx.handle, ctypes.byref(self.params), _lib.ptr(src),
                                                      _lib.ptr(soff), len(srcs), _lib.ptr(tgt), _lib.ptr(toff),
                                                      len(tgts), _lib.ptr(ids), _lib.ptr(ids), n, 3, _lib.ptr(g),
                                                      _lib.ptr(T), _lib.ptr(iters), _lib.ptr(inl), _lib.ptr(st)),
                       "ICP.compute_pairs")
        else:
            _lib.check(ctx.lib.sfe_icp_batch_host(ctx.handle, ctypes.byref(self.params), _lib.ptr(src), _lib.ptr(soff),
                                                  len(srcs), _lib.ptr(tgt), _lib.ptr(toff), len(tgts), _lib.ptr(ids),
                                                  _lib.ptr(ids), n, _lib.ptr(g), _lib.ptr(T), _lib.ptr(iters),
                                                  _lib.ptr(inl), _lib.ptr(st)), "ICP.compute_pairs")
        msgs = self._results(ctx, st)
        out, a = [], 0
        for c in counts:
            b = a + int(c)
            out.append(dict(messages=msgs[a:b], T=T[a:b], iterations=iters[a:b], inliers=inl[a:b], status=st[a:b]))
            a = b
        return out

    def getCovariance(self):
        raise NotImplementedError("ICP.getCovariance is never called by the reference's Python and is not provided")
