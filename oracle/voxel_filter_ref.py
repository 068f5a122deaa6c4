"""TEST INFRASTRUCTURE ONLY -- ctypes doorway onto oracle/voxel_filter_ref.c: libpointmatcher's
VoxelGridDataPointsFilter (useCentroid) as an ICP data filter, the data-filter chains that mix it with the octree and
distance filters, and the ICP restatement of oracle/icp_filters_ref.c behind those chains.

The library (voxel_filter_ref.c, which includes octree_filter_ref.c, icp_filters_ref.c and icp_ref.c, plus
cloud_ref.c's grid search) is compiled on first use with the flags of oracle/Makefile's restatements into
oracle/_build/libvoxel_filter_ref.so, or into a temporary directory when the tree is read-only, and rebuilt whenever one
of its sources is newer.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from .icp_filters_ref import CFLAGS, MAX_DIST, MIN_DIST, IcpFilters  # noqa: F401  (the same filter block)
from .octree_filter_ref import OCTREE  # noqa: F401
from .oracle import ICP_MESSAGES, IcpParams

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, f) for f in ("voxel_filter_ref.c", "cloud_ref.c")]
_DEPS = _SRCS + [os.path.join(_HERE, f) for f in ("octree_filter_ref.c", "icp_filters_ref.c", "icp_ref.c")]
VOXEL = 4  # data filter kind: dim = useCentroid (1), dist = vSize
_lib = None


class VoxelOverflow(ValueError):
    """A cloud's voxel grid has more than 2^32 - 1 voxels (or non-finite bounds): upstream's index would wrap."""


def _compile(out_dir):
    out = os.path.join(out_dir, "libvoxel_filter_ref.so")
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
        for f in ("orc_voxel_filter", "orc_chain_filters_voxel", "orc_icp_chain_voxel"):
            getattr(_lib, f).restype = ctypes.c_int
    return _lib


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def voxel_filter(pts, vsize):
    """VoxelGridDataPointsFilter {vSize, useCentroid 1} alone on pts [N,2] -> float32 [M,2]: the first point of every
    voxel, in input order, holding its voxel's centroid.  Raises VoxelOverflow when the index would not fit 32 bits."""
    lib = _load()
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    out = np.empty_like(pts)
    m = lib.orc_voxel_filter(_fp(pts), len(pts), ctypes.c_float(vsize), _fp(out))
    if m < 0:
        raise VoxelOverflow(f"voxel grid of vSize {vsize} over more than 2^32 - 1 voxels")
    return out[:m].copy()


def data_filters(pts, filters):
    """The data-filter chain [(kind, dim, dist), ...] (kinds MAX_DIST, MIN_DIST, OCTREE, VOXEL) on pts [N,2] -> the
    filtered cloud float32 [M,2].  Raises VoxelOverflow as voxel_filter."""
    lib = _load()
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    fl = IcpFilters(reading=filters)
    out = np.empty_like(pts)
    m = lib.orc_chain_filters_voxel(fl.reading, len(filters), _fp(pts), len(pts), _fp(out))
    if m < 0:
        raise VoxelOverflow("a voxel filter's grid has more than 2^32 - 1 voxels")
    return out[:m].copy()


def icp(src, tgt, guess=None, params=None, filters=None):
    """icp_filters_ref.icp with chains that may hold octree and voxel filters -> dict(message, T, iterations, inliers,
    status).  Raises VoxelOverflow as voxel_filter."""
    lib = _load()
    src = np.ascontiguousarray(src, np.float32).reshape(-1, 2)
    tgt = np.ascontiguousarray(tgt, np.float32).reshape(-1, 2)
    g = np.eye(3, dtype=np.float32) if guess is None else np.ascontiguousarray(guess, np.float32)
    prm = params or IcpParams()
    fl = filters or IcpFilters()
    T = np.empty((3, 3), np.float32)
    it, inl = ctypes.c_int(0), ctypes.c_int(0)
    st = lib.orc_icp_chain_voxel(_fp(src), len(src), _fp(tgt), len(tgt), _fp(g), ctypes.byref(prm), ctypes.byref(fl),
                                 _fp(T), ctypes.byref(it), ctypes.byref(inl))
    if st < 0:
        raise VoxelOverflow("a voxel filter's grid has more than 2^32 - 1 voxels")
    return dict(message=ICP_MESSAGES[st], status=st, T=T if st == 0 else g.copy(), iterations=it.value,
                inliers=inl.value)
