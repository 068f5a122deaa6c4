"""TEST INFRASTRUCTURE ONLY -- ctypes doorway onto oracle/octree_filter_ref.c: libpointmatcher's
OctreeGridDataPointsFilter as an ICP data filter, the data-filter chains that mix it with the distance filters, and the
ICP restatement of oracle/icp_filters_ref.c behind those chains.

The library (octree_filter_ref.c, which includes icp_filters_ref.c and icp_ref.c, plus cloud_ref.c's grid search) is
compiled on first use with the flags of oracle/Makefile's restatements into oracle/_build/liboctree_filter_ref.so, or
into a temporary directory when the tree is read-only, and rebuilt whenever one of its sources is newer.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from .icp_filters_ref import CFLAGS, MAX_DIST, MIN_DIST, IcpFilters  # noqa: F401  (the same filter block)
from .oracle import ICP_MESSAGES, IcpParams

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, f) for f in ("octree_filter_ref.c", "cloud_ref.c")]
_DEPS = _SRCS + [os.path.join(_HERE, f) for f in ("icp_filters_ref.c", "icp_ref.c")]
OCTREE = 3  # data filter kind: dim = samplingMethod (0 first point, 2 centroid, 3 medoid), dist = maxSizeByNode
_lib = None


def _compile(out_dir):
    out = os.path.join(out_dir, "liboctree_filter_ref.so")
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
        for f in ("orc_octree_filter", "orc_octree_filter_depth", "orc_chain_filters", "orc_icp_chain"):
            getattr(_lib, f).restype = ctypes.c_int
    return _lib


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def octree_filter(pts, max_size, sampler, max_depth=15):
    """OctreeGridDataPointsFilter {maxSizeByNode, samplingMethod} alone on pts [N,2] -> float32 [M,2] in leaf order;
    max_depth: the tree's cut (15 in an ICP chain, as on the device; None: no cut)."""
    lib = _load()
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    out = np.empty_like(pts)
    depth = 2 ** 31 - 1 if max_depth is None else int(max_depth)
    m = lib.orc_octree_filter_depth(_fp(pts), len(pts), ctypes.c_float(max_size), int(sampler), depth, _fp(out))
    return out[:m].copy()


def data_filters(pts, filters):
    """The data-filter chain [(kind, dim, dist), ...] (kinds MAX_DIST, MIN_DIST, OCTREE) on pts [N,2] -> the filtered
    cloud float32 [M,2]: the distance filters' survivors in their order, the octree filters' points in leaf order."""
    lib = _load()
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    fl = IcpFilters(reading=filters)
    out = np.empty_like(pts)
    m = lib.orc_chain_filters(fl.reading, len(filters), _fp(pts), len(pts), _fp(out))
    return out[:m].copy()


def icp(src, tgt, guess=None, params=None, filters=None):
    """icp_filters_ref.icp with chains that may hold octree filters -> dict(message, T, iterations, inliers,
    status)."""
    lib = _load()
    src = np.ascontiguousarray(src, np.float32).reshape(-1, 2)
    tgt = np.ascontiguousarray(tgt, np.float32).reshape(-1, 2)
    g = np.eye(3, dtype=np.float32) if guess is None else np.ascontiguousarray(guess, np.float32)
    prm = params or IcpParams()
    fl = filters or IcpFilters()
    T = np.empty((3, 3), np.float32)
    it, inl = ctypes.c_int(0), ctypes.c_int(0)
    st = lib.orc_icp_chain(_fp(src), len(src), _fp(tgt), len(tgt), _fp(g), ctypes.byref(prm), ctypes.byref(fl),
                           _fp(T), ctypes.byref(it), ctypes.byref(inl))
    return dict(message=ICP_MESSAGES[st], status=st, T=T if st == 0 else g.copy(), iterations=it.value,
                inliers=inl.value)
