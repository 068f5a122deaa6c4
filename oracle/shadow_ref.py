"""TEST INFRASTRUCTURE ONLY -- ctypes doorway onto oracle/shadow_ref.c: libpointmatcher's SurfaceNormalDataPointsFilter
and ShadowDataPointsFilter on the reading cloud, and the whole ICP chain with them -- the reading chain, then
oracle/sampling_normal_ref.c's reference chain and iterations.

The library (shadow_ref.c, which includes sampling_normal_ref.c, robust_ref.c, voxel_filter_ref.c, octree_filter_ref.c,
icp_filters_ref.c and icp_ref.c, plus cloud_ref.c's grid search) is compiled on first use with the flags of
oracle/Makefile's restatements into oracle/_build/libshadow_ref.so, or into a temporary directory when the tree is
read-only, and rebuilt whenever one of its sources is newer.
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
_SRCS = [os.path.join(_HERE, f) for f in ("shadow_ref.c", "cloud_ref.c")]
_DEPS = _SRCS + [os.path.join(_HERE, f) for f in ("sampling_normal_ref.c", "robust_ref.c", "voxel_filter_ref.c",
                                                  "octree_filter_ref.c", "icp_filters_ref.c", "icp_ref.c")]
NORMALS = 6  # reading data filter kind: dim = knn (3..16)
SHADOW = 7   # reading data filter kind: dist = eps (radians), after a NORMALS
_lib = None


def _compile(out_dir):
    out = os.path.join(out_dir, "libshadow_ref.so")
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
        for f in ("orc_chain_filters_shadow", "orc_icp_shadow", "orc_shadow_keep"):
            getattr(_lib, f).restype = ctypes.c_int
        _lib.orc_reading_normals.restype = None
        _lib.orc_reading_normals.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.c_int, ctypes.c_int,
                                             ctypes.POINTER(ctypes.c_float)]
        _lib.orc_shadow_keep.argtypes = [ctypes.c_float] * 5
        _lib.orc_sinf.restype = ctypes.c_float
        _lib.orc_sinf.argtypes = [ctypes.c_float]
    return _lib


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def reading_normals(pts, knn=5):
    """The reading SurfaceNormalDataPointsFilter's normals of pts [N,2] -> float32 [N,2], in point order."""
    lib = _load()
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    nrm = np.zeros_like(pts)
    lib.orc_reading_normals(_fp(pts), len(pts), int(knn), _fp(nrm))
    return nrm


def sin_eps(eps):
    """sinf(eps) of the C library, the threshold ShadowDataPointsFilter compares with."""
    return np.float32(_load().orc_sinf(float(eps)))


def shadow_keep(x, y, nx, ny, eps):
    """The shadow test of one point (x, y) with normal (nx, ny) -> bool."""
    return bool(_load().orc_shadow_keep(float(x), float(y), float(nx), float(ny), float(sin_eps(eps))))


def data_filters(pts, filters):
    """A reading chain [(kind, dim, dist), ...] that may hold NORMALS and SHADOW -> points [M,2].  Raises VoxelOverflow as
    voxel_filter_ref.data_filters."""
    lib = _load()
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    fl = IcpFilters(reading=filters)
    out = np.empty_like(pts)
    m = lib.orc_chain_filters_shadow(fl.reading, len(filters), _fp(pts), len(pts), _fp(out))
    if m < 0:
        raise VoxelOverflow("a voxel filter's grid has more than 2^32 - 1 voxels")
    return out[:m].copy()


def icp(src, tgt, guess=None, params=None, filters=None, robust=None):
    """sampling_normal_ref.icp with a reading chain that may hold NORMALS and SHADOW -> dict(message, T, iterations,
    inliers, status)."""
    lib = _load()
    src = np.ascontiguousarray(src, np.float32).reshape(-1, 2)
    tgt = np.ascontiguousarray(tgt, np.float32).reshape(-1, 2)
    g = np.eye(3, dtype=np.float32) if guess is None else np.ascontiguousarray(guess, np.float32)
    prm = params or IcpParams()
    fl = filters or IcpFilters()
    T = np.empty((3, 3), np.float32)
    it, inl = ctypes.c_int(0), ctypes.c_int(0)
    st = lib.orc_icp_shadow(_fp(src), len(src), _fp(tgt), len(tgt), _fp(g), ctypes.byref(prm), ctypes.byref(fl),
                            ctypes.byref(robust) if robust is not None else None, _fp(T), ctypes.byref(it),
                            ctypes.byref(inl))
    if st < 0:
        raise VoxelOverflow("a voxel filter's grid has more than 2^32 - 1 voxels")
    return dict(message=ICP_MESSAGES[st], status=st, T=T if st == 0 else g.copy(), iterations=it.value,
                inliers=inl.value)
