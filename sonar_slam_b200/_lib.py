"""ctypes binding of libsonarfe.so (the C ABI declared in include/sonarfe.h).

Fails loudly: a missing shared object or a machine without an H100 (sm_90) raises -- there
is no CPU path behind these functions.
"""
import ctypes
import os
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SFE_LIB_PATH") or os.path.join(_HERE, "libsonarfe.so")  # (override: kernel experiments)

c_int, c_double, c_void_p, c_float = ctypes.c_int, ctypes.c_double, ctypes.c_void_p, ctypes.c_float
MAX_GEOMETRIES = 8  # SFE_FE_MAX_GEOMETRIES: sonar geometries per front end, the creation maps included

_lib = None
_lock = threading.Lock()


class SonarFEError(RuntimeError):
    pass


ERR_CAPACITY = -3  # SFE_ERR_CAPACITY: a caller-provided output buffer was too small
ICP_SKIPPED, ICP_TOO_LARGE = 7, 8  # SFE_ICP_SKIPPED, SFE_ICP_TOO_LARGE


def load():
    """Load (building first if sources are newer and nvcc is present) and type the library."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            from . import build as _build
            _build.build()
        if not os.path.exists(LIB_PATH):
            raise SonarFEError(f"{LIB_PATH} is missing: build it with `python -m sonar_slam_b200.build`")
        lib = ctypes.CDLL(LIB_PATH)
        lib.sfe_version.restype = c_int
        lib.sfe_last_error.restype = ctypes.c_char_p
        lib.sfe_ctx_create.argtypes = [c_int, c_void_p, c_int, ctypes.POINTER(c_void_p)]
        lib.sfe_ctx_destroy.argtypes = [c_void_p]
        lib.sfe_ctx_destroy.restype = None
        lib.sfe_sync.argtypes = [c_void_p]
        lib.sfe_launch_count.argtypes = [c_void_p]
        lib.sfe_launch_count.restype = ctypes.c_uint64
        cfar_args = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_double,
                     c_int, c_double, c_void_p, c_void_p]
        lib.sfe_cfar_dev.argtypes = cfar_args + [c_void_p]
        lib.sfe_cfar_host.argtypes = cfar_args
        _type_more(lib)
        lib.sfe_maps_destroy.argtypes = [c_void_p]
        lib.sfe_maps_destroy.restype = None
        lib.sfe_costmap_destroy.argtypes = [c_void_p]
        lib.sfe_costmap_destroy.restype = None
        lib.sfe_keyframe_map_destroy.argtypes = [c_void_p]
        lib.sfe_keyframe_map_destroy.restype = None
        lib.sfe_icp_status_message.argtypes = [c_int]
        lib.sfe_icp_status_message.restype = ctypes.c_char_p
        lib.sfe_icp_params_default.argtypes = [c_void_p]
        lib.sfe_icp_params_default.restype = None
        lib.sfe_frontend_params_default.argtypes = [c_void_p]
        lib.sfe_frontend_params_default.restype = None
        lib.sfe_frontend_destroy.argtypes = [c_void_p]
        lib.sfe_frontend_destroy.restype = None
        lib.sfe_jpeg_status_message.argtypes = [c_int]
        lib.sfe_jpeg_status_message.restype = ctypes.c_char_p
        lib.sfe_png_status_message.argtypes = [c_int]
        lib.sfe_png_status_message.restype = ctypes.c_char_p
        _lib = lib
        return lib


def _type_more(lib):
    """argtypes of the entry points added after the CFAR milestone (kept in one place)."""
    for name, args in _EXTRA_SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = c_int


_EXTRA_SIGNATURES = {
    "sfe_maps_inverse_lists_host": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                    ctypes.c_int64, ctypes.POINTER(ctypes.c_int64)],
    "sfe_costmap_create": [c_void_p, c_void_p, c_int, c_float, c_float, c_float, c_int, c_int, c_int, c_void_p,
                           c_void_p, ctypes.POINTER(c_void_p)],
    "sfe_costmap_grid_host": [c_void_p, c_void_p, c_void_p],
    "sfe_costmap_set_source_host": [c_void_p, c_void_p, c_void_p, c_int],
    "sfe_costmap_score_host": [c_void_p, c_void_p, c_void_p, c_int, c_void_p],
    "sfe_costmap_score_dev": [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p],
    "sfe_maps_create": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_double, c_double,
                        ctypes.POINTER(c_void_p)],
    "sfe_cart_points_dev": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "sfe_cart_points_host": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "sfe_downsample_dev": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p],
    "sfe_remove_outlier_dev": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_double, c_int, c_void_p, c_void_p,
                               c_void_p],
    "sfe_downsample_frames_dev": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p,
                                  c_void_p, c_void_p],
    "sfe_downsample_host": [c_void_p, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p],
    "sfe_downsample_cta_limit": [c_void_p, c_int, c_void_p],
    "sfe_remove_outlier_host": [c_void_p, c_void_p, c_int, c_int, c_double, c_int, c_void_p, c_void_p, c_void_p],
    "sfe_match_dev": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p],
    "sfe_match_host": [c_void_p, c_void_p, c_int, c_void_p, c_int, c_float, c_void_p, c_void_p],
    "sfe_match_knn_dev": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p,
                          c_void_p],
    "sfe_match_knn_host": [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p],
    "sfe_match_dim_dev": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p,
                          c_void_p],
    "sfe_match_dim_host": [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p],
    "sfe_match_knn_dim_dev": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float,
                              c_void_p, c_void_p],
    "sfe_match_knn_dim_host": [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p],
    "sfe_icp_dev": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                    c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sfe_frontend_icp_dev": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sfe_copy_to_host": [c_void_p, c_void_p, c_void_p, ctypes.c_uint64],
    "sfe_ctx_set_grid_sms": [c_void_p, c_int, ctypes.POINTER(ctypes.c_int32)],
    "sfe_ctx_occupancy": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, ctypes.POINTER(ctypes.c_int32)],
    "sfe_frontend_create": [c_void_p, c_void_p, c_void_p, c_int, ctypes.POINTER(c_void_p)],
    "sfe_frontend_set_timing": [c_void_p, c_int],
    "sfe_frontend_set_carry": [c_void_p, c_int],
    "sfe_frontend_set_clouds": [c_void_p, c_void_p, ctypes.c_int64, c_void_p, c_int],
    "sfe_frontend_set_scan_match": [c_void_p, c_int],
    "sfe_frontend_get_timing": [c_void_p, c_void_p, c_void_p],
    "sfe_frontend_run_dev": [c_void_p, c_void_p, c_void_p, c_int],
    "sfe_frontend_results_dev": [c_void_p] + [ctypes.POINTER(c_void_p)] * 6 + [ctypes.POINTER(ctypes.c_int32)],
    "sfe_frontend_run_host": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                              c_void_p],
    "sfe_fov_select_dev": [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p],
    "sfe_fov_select_host": [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p],
    "sfe_keyframe_map_create": [c_void_p, c_int, ctypes.POINTER(c_void_p)],
    "sfe_keyframe_map_size": [c_void_p, ctypes.POINTER(c_int), ctypes.POINTER(ctypes.c_int64)],
    "sfe_keyframe_map_append_host": [c_void_p, c_void_p, c_void_p, c_int, c_void_p],
    "sfe_keyframe_map_append_dev": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p],
    "sfe_keyframe_map_assemble_dev": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_int, c_void_p,
                                      c_void_p, c_void_p],
    "sfe_keyframe_map_assemble_host": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_int, c_void_p,
                                       c_void_p, c_void_p],
    "sfe_icp_host": [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p,
                     c_void_p, c_void_p],
    "sfe_icp_batch_host": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p,
                           c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sfe_icp_set_filters": [c_void_p, c_void_p],
    "sfe_icp_dim_dev": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                        c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sfe_icp_dim_host": [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p,
                         c_void_p, c_void_p, c_void_p],
    "sfe_icp_batch_dim_host": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p,
                               c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sfe_icp_cta_limit": [c_void_p, c_int, c_int, c_void_p],
    "sfe_icp_sampling_normals_dev": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p,
                                     c_void_p, c_void_p],
    "sfe_icp_surface_normals_dev": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "sfe_icp_source_limit": [c_void_p, c_void_p, c_int, c_void_p],
    "sfe_frontend_set_icp_filters": [c_void_p, c_void_p],
    "sfe_icp_set_robust": [c_void_p, c_void_p],
    "sfe_frontend_set_icp_robust": [c_void_p, c_void_p],
    "sfe_mincovdet_dev": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_double, c_double, c_int,
                          c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sfe_mincovdet_host": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_double, c_double, c_int,
                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sfe_jpeg_inspect_host": [c_void_p, c_void_p, c_int, c_void_p],
    "sfe_jpeg_decode_host": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "sfe_jpeg_decode_to_dev": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "sfe_jpeg_coefficients_host": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p],
    "sfe_jpeg_set_timing": [c_void_p, c_int],
    "sfe_jpeg_get_timing": [c_void_p, c_void_p, c_void_p],
    "sfe_frontend_run_jpeg_host": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p],
    "sfe_png_inspect_host": [c_void_p, c_void_p, c_int, c_void_p],
    "sfe_png_decode_host": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "sfe_png_decode_to_dev": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "sfe_png_set_timing": [c_void_p, c_int],
    "sfe_png_get_timing": [c_void_p, c_void_p, c_void_p],
    "sfe_frontend_run_png_host": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p],
    "sfe_feature_image_dev": [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p],
    "sfe_feature_image_host": [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p],
    "sfe_frontend_set_feature_images": [c_void_p, c_void_p, c_void_p, c_int],
    "sfe_frontend_add_geometry": [c_void_p, c_void_p, ctypes.POINTER(c_int)],
    "sfe_frontend_run_dev_geometry": [c_void_p, c_void_p, c_void_p, c_void_p, c_int],
    "sfe_frontend_run_host_geometry": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                       c_void_p, c_void_p, c_void_p, c_void_p],
    "sfe_frontend_run_jpeg_host_geometry": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                            c_void_p, c_void_p, c_void_p, c_void_p],
    "sfe_frontend_run_png_host_geometry": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p],
}


class FrontendParams(ctypes.Structure):
    """sfe_frontend_params (include/sonarfe.h)."""
    pass


class IcpParams(ctypes.Structure):
    """sfe_icp_params (include/sonarfe.h); defaults = bruce_slam/config/icp.yaml."""
    _fields_ = [("matcher_max_dist", c_float), ("outlier_max_dist", c_float), ("trim_ratio", c_float),
                ("max_iterations", c_int), ("min_diff_rot", c_float), ("min_diff_trans", c_float),
                ("smooth_length", c_int), ("flags", c_int), ("minimizer", c_int), ("normals_knn", c_int)]

    def __init__(self, matcher_max_dist=10.0, outlier_max_dist=3.0, trim_ratio=0.8, max_iterations=40,
                 min_diff_rot=0.01, min_diff_trans=0.1, smooth_length=4, flags=0, minimizer=0, normals_knn=5):
        super().__init__(matcher_max_dist, outlier_max_dist, trim_ratio, max_iterations, min_diff_rot,
                         min_diff_trans, smooth_length, flags, minimizer, normals_knn)


MAX_DIST, MIN_DIST = 1, 2  # SFE_ICP_DATA_MAX_DIST, SFE_ICP_DATA_MIN_DIST: the kinds of an IcpDataFilter
OCTREE = 3                 # SFE_ICP_DATA_OCTREE: OctreeGridDataPointsFilter {dim samplingMethod, dist maxSizeByNode}
VOXEL = 4                  # SFE_ICP_DATA_VOXEL: VoxelGridDataPointsFilter {dim useCentroid (1), dist vSize}
SAMPLING_NORMALS = 5       # SFE_ICP_DATA_SAMPLING_NORMALS: SamplingSurfaceNormalDataPointsFilter {dim samplingMethod,
                           # dist maxBoxDim}; its knn is IcpParams.normals_knn
NORMALS = 6                # SFE_ICP_DATA_NORMALS: SurfaceNormalDataPointsFilter on the reading {dim knn (3..16)}
SHADOW = 7                 # SFE_ICP_DATA_SHADOW: ShadowDataPointsFilter on the reading {dist eps}, after a NORMALS
MAX_DATA_FILTERS = 4       # SFE_ICP_MAX_DATA_FILTERS per cloud


class IcpDataFilter(ctypes.Structure):
    """sfe_icp_data_filter: MaxDist / MinDistDataPointsFilter {dim, dist}, OctreeGridDataPointsFilter {dim =
    samplingMethod (0 first point, 2 centroid, 3 medoid), dist = maxSizeByNode}, or VoxelGridDataPointsFilter {dim =
    useCentroid (1), dist = vSize}."""
    _fields_ = [("kind", c_int), ("dim", c_int), ("dist", c_float)]


class IcpFilters(ctypes.Structure):
    """sfe_icp_filters (include/sonarfe.h): the MinDist / MedianDist outlier filters (< 0: off) and up to four data
    filters per cloud, run in their order.  reading / reference: sequences of (kind, dim, dist): kind MAX_DIST or
    MIN_DIST with dim -1 (radial), 0 (x) or 1 (y) and the distance; kind OCTREE with dim the samplingMethod (0 first
    point, 2 centroid, 3 medoid) and dist maxSizeByNode (finite, > 0); kind VOXEL with dim 1 (useCentroid) and dist
    vSize (finite, > 0); kind SAMPLING_NORMALS (reference, last); on the reading, kind NORMALS with dim the knn (3..16)
    and kind SHADOW with dist eps (finite), after a NORMALS that only distance filters and SHADOW follow."""
    _fields_ = [("min_dist", c_float), ("median_factor", c_float), ("n_reading", c_int), ("n_reference", c_int),
                ("reading", IcpDataFilter * MAX_DATA_FILTERS), ("reference", IcpDataFilter * MAX_DATA_FILTERS)]

    def __init__(self, min_dist=-1.0, median_factor=-1.0, reading=(), reference=()):
        if len(reading) > MAX_DATA_FILTERS or len(reference) > MAX_DATA_FILTERS:
            raise ValueError(f"IcpFilters: at most {MAX_DATA_FILTERS} data filters per cloud")
        super().__init__(min_dist, median_factor, len(reading), len(reference))
        for arr, fl in ((self.reading, reading), (self.reference, reference)):
            for k, (kind, dim, dist) in enumerate(fl):
                arr[k] = IcpDataFilter(int(kind), int(dim), float(dist))

    def data_filters(self, which):
        """[(kind, dim, dist), ...] of 'reading' or 'reference'."""
        arr, n = (self.reading, self.n_reading) if which == "reading" else (self.reference, self.n_reference)
        return [(arr[k].kind, arr[k].dim, arr[k].dist) for k in range(n)]


# SFE_ICP_ROBUST_*: RobustOutlierFilter robustFct codes
ROBUST_FCT = {"cauchy": 1, "welsch": 2, "sc": 3, "gm": 4, "tukey": 5, "huber": 6, "L1": 7}


class IcpRobust(ctypes.Structure):
    """sfe_icp_robust (include/sonarfe.h): libpointmatcher's RobustOutlierFilter with scaleEstimator none / fixed --
    fct a ROBUST_FCT name or code, tuning k (finite, > 0), approximation (weight 0 where the squared distance is at
    least this; +inf: no cut-off)."""
    _fields_ = [("fct", c_int), ("tuning", c_float), ("approximation", c_float)]

    def __init__(self, fct="cauchy", tuning=1.0, approximation=float("inf")):
        super().__init__(ROBUST_FCT[fct] if isinstance(fct, str) else int(fct), float(tuning), float(approximation))


class IcpConfig(IcpParams):
    """IcpParams as an ICP YAML configures it (bruce_slam.pcl.parse_icp_yaml): the same structure, passed by reference
    where IcpParams is, plus `.filters` -- the IcpFilters of the modules IcpParams does not carry, or None -- and
    `.robust` -- the IcpRobust of a RobustOutlierFilter, or None."""

    def __init__(self, *args, filters=None, robust=None, **kwargs):
        super().__init__(*args, **kwargs)
        self.filters = filters
        self.robust = robust


def icp_filters_of(params, filters=None):
    """The filters a call with these ICP parameters runs: `filters` when given, else params.filters (IcpConfig)."""
    return filters if filters is not None else getattr(params, "filters", None)


def set_icp_filters(ctx, filters):
    """sfe_icp_set_filters on ctx (None: no filter), so a call never inherits an earlier call's filters."""
    check(ctx.lib.sfe_icp_set_filters(ctx.handle, ctypes.byref(filters) if filters is not None else None),
          "sfe_icp_set_filters")


def icp_robust_of(params, robust=None):
    """The RobustOutlierFilter a call with these ICP parameters runs: `robust` when given, else params.robust
    (IcpConfig)."""
    return robust if robust is not None else getattr(params, "robust", None)


def set_icp_robust(ctx, robust):
    """sfe_icp_set_robust on ctx (None: no robust filter), so a call never inherits an earlier call's setting."""
    check(ctx.lib.sfe_icp_set_robust(ctx.handle, ctypes.byref(robust) if robust is not None else None),
          "sfe_icp_set_robust")


FrontendParams._fields_ = [
    ("R", c_int), ("B", c_int), ("cfar_alg", c_int), ("train_hs", c_int), ("guard_hs", c_int), ("rank", c_int),
    ("tau", c_double), ("gate_enable", c_int), ("gate_threshold", c_double), ("resolution", c_float),
    ("outlier_radius", c_double), ("outlier_min_points", c_int), ("window", c_int), ("submap_resolution", c_float),
    ("min_points", c_int), ("icp", IcpParams), ("cap_points", c_int), ("cap_source", c_int), ("cap_target", c_int), ("flip_lateral", c_int)]


def check(rc, what=""):
    if rc != 0:
        msg = load().sfe_last_error().decode(errors="replace")
        raise SonarFEError(f"{what or 'libsonarfe'} failed (code {rc}): {msg}")


class Context:
    """One GPU + one stream + scratch (sfe_ctx).  Not thread-safe; make one per thread."""

    def __init__(self, device=0, stream="own"):
        """stream: "own" -> library-owned stream; otherwise a cudaStream_t integer handle of the
        caller (0 / None = the legacy default stream, e.g. torch.cuda.current_stream().cuda_stream)."""
        self.lib = load()
        h = c_void_p()
        own = 1 if stream == "own" else 0
        sp = None if (own or not stream) else c_void_p(int(stream))
        check(self.lib.sfe_ctx_create(int(device), sp, own, ctypes.byref(h)), "sfe_ctx_create")
        self.handle = h
        self.device = int(device)

    def sync(self):
        check(self.lib.sfe_sync(self.handle), "sfe_sync")

    def to_host(self, dev_ptr, shape, dtype):
        """Blocking copy of a device buffer (raw address) into a new numpy array."""
        out = np.empty(shape, dtype)
        check(self.lib.sfe_copy_to_host(self.handle, ptr(out), c_void_p(int(dev_ptr)), out.nbytes), "sfe_copy_to_host")
        return out

    @property
    def launches(self):
        return int(self.lib.sfe_launch_count(self.handle))

    def set_grid_sms(self, n):
        """For tests: size this context's persistent launches for min(n, the device's) SMs (n <= 0: the device's
        count), so that each CTA takes more work items in a row; results do not change (sfe_ctx_set_grid_sms).
        Returns the count now in force."""
        eff = ctypes.c_int32()
        check(self.lib.sfe_ctx_set_grid_sms(self.handle, int(n), ctypes.byref(eff)), "sfe_ctx_set_grid_sms")
        return eff.value

    def occupancy(self):
        """For tests: [(threads, dynamic shared memory bytes, CTAs per SM), ...] of the persistent one-CTA launch
        configurations this context has sized, oldest first (the last 16; sfe_ctx_occupancy)."""
        cap = 16
        t, s, q = (np.zeros(cap, np.int32) for _ in range(3))
        n = ctypes.c_int32()
        check(self.lib.sfe_ctx_occupancy(self.handle, ptr(t), ptr(s), ptr(q), cap, ctypes.byref(n)),
              "sfe_ctx_occupancy")
        return [(int(t[k]), int(s[k]), int(q[k])) for k in range(min(n.value, cap))]

    def close(self):
        if getattr(self, "handle", None):
            self.lib.sfe_ctx_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_ctx = {}


def default_context(device=0):
    """Process-wide context used by the drop-in single-call API (bruce_slam.cfar / .pcl)."""
    key = (os.getpid(), threading.get_ident(), int(device))
    ctx = _default_ctx.get(key)
    if ctx is None:
        ctx = _default_ctx[key] = Context(device)
    return ctx


class Maps:
    """Device-resident polar->Cartesian sampling table for one sonar geometry (sfe_maps); a FrontEnd may hold several
    (FrontEnd.add_geometry)."""

    def __init__(self, ctx, map_x, map_y, R, B, width, height):
        map_x = np.ascontiguousarray(map_x, np.float32)
        map_y = np.ascontiguousarray(map_y, np.float32)
        if map_x.shape != map_y.shape or map_x.ndim != 2:
            raise ValueError("map_x / map_y must be 2-D arrays of the same shape")
        self.rows, self.cols = map_x.shape
        self.R, self.B = int(R), int(B)
        self.width, self.height = float(width), float(height)
        self.lib = ctx.lib
        h = c_void_p()
        check(ctx.lib.sfe_maps_create(ctx.handle, ptr(map_x), ptr(map_y), self.rows, self.cols, self.R, self.B,
                                      self.width, self.height, ctypes.byref(h)), "sfe_maps_create")
        self.handle = h

    def close(self):
        if getattr(self, "handle", None):
            self.lib.sfe_maps_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def inverse_lists(map_x, map_y, R, B):
    """Host-only diagnostic (no GPU needed): the CSR inverse lists (polar cell -> Cartesian pixels to test) that
    sfe_maps_create uploads for these sampling maps.  Returns (off int32 [R*B+1], idx int32 [n])."""
    lib = load()
    map_x = np.ascontiguousarray(map_x, np.float32)
    map_y = np.ascontiguousarray(map_y, np.float32)
    rows, cols = map_x.shape
    off = np.empty(R * B + 1, np.int32)
    cap = 4 * rows * cols
    idx = np.empty(cap, np.int32)
    n = ctypes.c_int64(0)
    check(lib.sfe_maps_inverse_lists_host(ptr(map_x), ptr(map_y), rows, cols, int(R), int(B), ptr(off), ptr(idx), cap,
                                          ctypes.byref(n)), "sfe_maps_inverse_lists_host")
    return off, idx[: n.value].copy()


def ellipse_spans(hs):
    """Column spans [lo, hi) per row of cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (2*hs+1, 2*hs+1), (hs, hs))
    (OpenCV's formula: dx = cvRound(c * sqrt((r*r - dy*dy) / (r*r))), columns c-dx .. c+dx); checked against
    cv2 itself in tests/test_oracle_globalinit.py."""
    k = 2 * int(hs) + 1
    r = c = k // 2
    inv_r2 = 1.0 / (r * r) if r else 0.0
    lo, hi = np.zeros(k, np.int32), np.zeros(k, np.int32)
    for i in range(k):
        dy = i - r
        dx = int(np.rint(c * np.sqrt((r * r - dy * dy) * inv_r2)))
        lo[i], hi[i] = max(c - dx, 0), min(c + dx + 1, k)
    return lo, hi


class CostMap:
    """Dilated occupancy grid of a target cloud on the device + candidate-pose scoring (sfe_costmap);
    the state behind the closure of SLAM.get_matching_cost_subroutine1 (slam.py:461-570)."""

    def __init__(self, ctx, target_points, xmin, ymin, resolution, rows, cols, dilate_hs, se_lo=None, se_hi=None):
        tgt = np.ascontiguousarray(target_points, np.float32)
        if tgt.ndim != 2 or tgt.shape[1] != 2:
            raise ValueError("target_points must be [N, 2]")
        if se_lo is None:
            se_lo, se_hi = ellipse_spans(dilate_hs)
        se_lo = np.ascontiguousarray(se_lo, np.int32)
        se_hi = np.ascontiguousarray(se_hi, np.int32)
        if len(se_lo) != 2 * dilate_hs + 1 or len(se_hi) != len(se_lo):
            raise ValueError("structuring element needs 2*dilate_hs+1 row spans")
        self.ctx, self.lib = ctx, ctx.lib
        self.rows, self.cols = int(rows), int(cols)
        h = c_void_p()
        check(ctx.lib.sfe_costmap_create(ctx.handle, ptr(tgt), len(tgt), float(xmin), float(ymin), float(resolution),
                                         self.rows, self.cols, int(dilate_hs), ptr(se_lo), ptr(se_hi),
                                         ctypes.byref(h)), "sfe_costmap_create")
        self.handle = h

    def grid(self):
        out = np.empty((self.rows, self.cols), np.uint8)
        check(self.lib.sfe_costmap_grid_host(self.ctx.handle, self.handle, ptr(out)), "sfe_costmap_grid_host")
        return out

    def set_source(self, source_points):
        src = np.ascontiguousarray(source_points, np.float32)
        if src.ndim != 2 or src.shape[1] != 2:
            raise ValueError("source_points must be [N, 2]")
        check(self.lib.sfe_costmap_set_source_host(self.ctx.handle, self.handle, ptr(src), len(src)),
              "sfe_costmap_set_source_host")

    def score(self, transforms):
        """transforms: [K, 6] float32 rows (r00, r01, r10, r11, tx, ty) -> int32 [K] costs."""
        tf = np.ascontiguousarray(transforms, np.float32).reshape(-1, 6)
        cost = np.empty(len(tf), np.int32)
        check(self.lib.sfe_costmap_score_host(self.ctx.handle, self.handle, ptr(tf), len(tf), ptr(cost)),
              "sfe_costmap_score_host")
        return cost

    def score_dev(self, source_dev_ptr, n_source, transforms_dev_ptr, n_candidates, cost_dev_ptr, ctx=None):
        """Asynchronous on the stream of `ctx` (default: the context the map was built with)."""
        check(self.lib.sfe_costmap_score_dev((ctx or self.ctx).handle, self.handle, c_void_p(source_dev_ptr), int(n_source),
                                             c_void_p(transforms_dev_ptr), int(n_candidates), c_void_p(cost_dev_ptr)),
              "sfe_costmap_score_dev")

    def close(self):
        if getattr(self, "handle", None):
            self.lib.sfe_costmap_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def ptr(a):
    """Host pointer of a C-contiguous numpy array (or None)."""
    if a is None:
        return None
    assert isinstance(a, np.ndarray) and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_void_p)
