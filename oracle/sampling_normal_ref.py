"""TEST INFRASTRUCTURE ONLY -- ctypes doorway onto oracle/sampling_normal_ref.c: libpointmatcher's
SamplingSurfaceNormalDataPointsFilter (samplingMethod 1, or 0 with ratio 1) as the last reference data filter, and the
whole ICP chain with it -- the data filters of oracle/voxel_filter_ref.c, the filter, then the iterations of
oracle/robust_ref.c reading the filter's normals.

The library (sampling_normal_ref.c, which includes robust_ref.c, voxel_filter_ref.c, octree_filter_ref.c,
icp_filters_ref.c and icp_ref.c, plus cloud_ref.c's grid search) is compiled on first use with the flags of
oracle/Makefile's restatements into oracle/_build/libsampling_normal_ref.so, or into a temporary directory when the tree
is read-only, and rebuilt whenever one of its sources is newer.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from .icp_filters_ref import CFLAGS, IcpFilters
from .oracle import ICP_MESSAGES, IcpParams
from .voxel_filter_ref import VoxelOverflow

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, f) for f in ("sampling_normal_ref.c", "cloud_ref.c")]
_DEPS = _SRCS + [os.path.join(_HERE, f) for f in ("robust_ref.c", "voxel_filter_ref.c", "octree_filter_ref.c",
                                                  "icp_filters_ref.c", "icp_ref.c")]
SAMPLING_NORMALS = 5  # data filter kind: dim = samplingMethod (0 or 1), dist = maxBoxDim; knn = IcpParams.normals_knn
_lib = None


def _compile(out_dir):
    out = os.path.join(out_dir, "libsampling_normal_ref.so")
    if os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(s) for s in _DEPS):
        return out
    os.makedirs(out_dir, exist_ok=True)
    tmp = f"{out}.{os.getpid()}.tmp"
    subprocess.run([os.environ.get("CC", "gcc")] + CFLAGS + _SRCS + ["-lm", "-o", tmp], check=True)
    os.replace(tmp, out)  # atomic: a concurrent loader sees the old library or the new one
    return out


def _load():
    global _lib
    if _lib is None:
        try:
            path = _compile(os.path.join(_HERE, "_build"))
        except (OSError, subprocess.CalledProcessError):  # a read-only tree
            path = _compile(os.path.join(tempfile.gettempdir(), f"sonarfe_oracle_{os.getuid()}"))
        _lib = ctypes.CDLL(path)
        for f in ("orc_sampling_normals", "orc_chain_filters_sampling", "orc_icp_sampling"):
            getattr(_lib, f).restype = ctypes.c_int
        _lib.orc_sampling_normals.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                              ctypes.c_float, ctypes.POINTER(ctypes.c_float),
                                              ctypes.POINTER(ctypes.c_float)]
    return _lib


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def sampling_normals(pts, knn=7, method=1, max_box=float("inf")):
    """The filter alone on pts [N,2] -> (points float32 [M,2], normals float32 [M,2]), kept points in ascending index."""
    lib = _load()
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    out, nrm = np.empty_like(pts), np.empty_like(pts)
    m = lib.orc_sampling_normals(_fp(pts), len(pts), int(knn), int(method), float(max_box), _fp(out), _fp(nrm))
    return out[:m].copy(), nrm[:m].copy()


def data_filters(pts, filters, knn=7):
    """A reference chain [(kind, dim, dist), ...] that may end with SAMPLING_NORMALS -> (points [M,2], normals [M,2] or
    None when the chain has no such filter).  Raises VoxelOverflow as voxel_filter_ref.data_filters."""
    lib = _load()
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    fl = IcpFilters(reference=filters)
    out, nrm = np.empty_like(pts), np.empty_like(pts)
    has = ctypes.c_int(0)
    m = lib.orc_chain_filters_sampling(fl.reference, len(filters), _fp(pts), len(pts), int(knn), _fp(out), _fp(nrm),
                                       ctypes.byref(has))
    if m < 0:
        raise VoxelOverflow("a voxel filter's grid has more than 2^32 - 1 voxels")
    return out[:m].copy(), (nrm[:m].copy() if has.value else None)


def icp(src, tgt, guess=None, params=None, filters=None, robust=None):
    """robust_ref.icp with a reference chain that may end with SAMPLING_NORMALS (point-to-plane then reads its
    normals) -> dict(message, T, iterations, inliers, status)."""
    lib = _load()
    src = np.ascontiguousarray(src, np.float32).reshape(-1, 2)
    tgt = np.ascontiguousarray(tgt, np.float32).reshape(-1, 2)
    g = np.eye(3, dtype=np.float32) if guess is None else np.ascontiguousarray(guess, np.float32)
    prm = params or IcpParams()
    fl = filters or IcpFilters()
    T = np.empty((3, 3), np.float32)
    it, inl = ctypes.c_int(0), ctypes.c_int(0)
    st = lib.orc_icp_sampling(_fp(src), len(src), _fp(tgt), len(tgt), _fp(g), ctypes.byref(prm), ctypes.byref(fl),
                              ctypes.byref(robust) if robust is not None else None, _fp(T), ctypes.byref(it),
                              ctypes.byref(inl))
    if st < 0:
        raise VoxelOverflow("a voxel filter's grid has more than 2^32 - 1 voxels")
    return dict(message=ICP_MESSAGES[st], status=st, T=T if st == 0 else g.copy(), iterations=it.value,
                inliers=inl.value)
