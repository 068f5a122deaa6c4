"""TEST INFRASTRUCTURE ONLY -- ctypes doorway onto oracle/robust_ref.c: libpointmatcher's RobustOutlierFilter
(scaleEstimator none / fixed, point2point residuals) and the whole ICP chain with it -- the data filters of
oracle/voxel_filter_ref.c, then the weighted iterations.

The library (robust_ref.c, which includes voxel_filter_ref.c, octree_filter_ref.c, icp_filters_ref.c and icp_ref.c,
plus cloud_ref.c's grid search) is compiled on first use with the flags of oracle/Makefile's restatements into
oracle/_build/librobust_ref.so, or into a temporary directory when the tree is read-only, and rebuilt whenever one of its
sources is newer.
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
_SRCS = [os.path.join(_HERE, f) for f in ("robust_ref.c", "cloud_ref.c")]
_DEPS = _SRCS + [os.path.join(_HERE, f) for f in ("voxel_filter_ref.c", "octree_filter_ref.c", "icp_filters_ref.c",
                                                  "icp_ref.c")]
# robustFct codes (orc_robust.fct)
FCT = {"cauchy": 1, "welsch": 2, "sc": 3, "gm": 4, "tukey": 5, "huber": 6, "L1": 7}
_lib = None


class Robust(ctypes.Structure):
    """Mirror of orc_robust: fct (FCT), tuning k, approximation (weight 0 where e2 >= it)."""
    _fields_ = [("fct", ctypes.c_int), ("tuning", ctypes.c_float), ("approximation", ctypes.c_float)]

    def __init__(self, fct="cauchy", tuning=1.0, approximation=float("inf")):
        super().__init__(FCT[fct] if isinstance(fct, str) else int(fct), tuning, approximation)


def _compile(out_dir):
    out = os.path.join(out_dir, "librobust_ref.so")
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
        _lib.orc_icp_robust.restype = ctypes.c_int
        _lib.orc_robust_weight.restype = ctypes.c_float
        _lib.orc_robust_weight.argtypes = [ctypes.POINTER(Robust), ctypes.c_float]
    return _lib


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def weights(e2, robust):
    """The RobustOutlierFilter weights of squared distances e2 (float32 [N]) -> float32 [N]."""
    lib = _load()
    e2 = np.ascontiguousarray(e2, np.float32).reshape(-1)
    w = np.empty_like(e2)
    lib.orc_robust_weights(ctypes.byref(robust), _fp(e2), len(e2), _fp(w))
    return w


def icp(src, tgt, guess=None, params=None, filters=None, robust=None):
    """The chain: data filters, then ICP with the outlier filters' product weights -> dict(message, T, iterations,
    inliers, status).  robust None: no RobustOutlierFilter (then voxel_filter_ref.icp's results).  Raises
    VoxelOverflow as voxel_filter_ref.icp."""
    lib = _load()
    src = np.ascontiguousarray(src, np.float32).reshape(-1, 2)
    tgt = np.ascontiguousarray(tgt, np.float32).reshape(-1, 2)
    g = np.eye(3, dtype=np.float32) if guess is None else np.ascontiguousarray(guess, np.float32)
    prm = params or IcpParams()
    fl = filters or IcpFilters()
    T = np.empty((3, 3), np.float32)
    it, inl = ctypes.c_int(0), ctypes.c_int(0)
    st = lib.orc_icp_robust(_fp(src), len(src), _fp(tgt), len(tgt), _fp(g), ctypes.byref(prm), ctypes.byref(fl),
                            ctypes.byref(robust) if robust is not None else None, _fp(T), ctypes.byref(it),
                            ctypes.byref(inl))
    if st < 0:
        raise VoxelOverflow("a voxel filter's grid has more than 2^32 - 1 voxels")
    return dict(message=ICP_MESSAGES[st], status=st, T=T if st == 0 else g.copy(), iterations=it.value,
                inliers=inl.value)
