"""TEST INFRASTRUCTURE ONLY -- ctypes doorway onto oracle/icp_filters_ref.c: the ICP restatement with the distance data
filters and the MinDist / MedianDist outlier filters.

The library (icp_filters_ref.c, which includes icp_ref.c, plus cloud_ref.c's grid search) is compiled on first use with
the flags of oracle/Makefile's restatements into oracle/_build/libicp_filters_ref.so, or into a temporary directory when
the tree is read-only, and rebuilt whenever one of its sources is newer.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from .oracle import ICP_MESSAGES, IcpParams

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, f) for f in ("icp_filters_ref.c", "cloud_ref.c")]
_DEPS = _SRCS + [os.path.join(_HERE, "icp_ref.c")]
CFLAGS = ["-O3", "-std=c11", "-fPIC", "-ffp-contract=off", "-Wall", "-Wextra", "-shared"]
MAX_DIST, MIN_DIST = 1, 2  # data filter kinds
MAX_DATA_FILTERS = 4
_lib = None


class DataFilter(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_int), ("dim", ctypes.c_int), ("dist", ctypes.c_float)]


class IcpFilters(ctypes.Structure):
    """Mirror of orc_icp_filters.  reading / reference: sequences of (kind, dim, dist), kind MAX_DIST or MIN_DIST."""
    _fields_ = [("min_dist", ctypes.c_float), ("median_factor", ctypes.c_float), ("n_reading", ctypes.c_int),
                ("n_reference", ctypes.c_int), ("reading", DataFilter * MAX_DATA_FILTERS),
                ("reference", DataFilter * MAX_DATA_FILTERS)]

    def __init__(self, min_dist=-1.0, median_factor=-1.0, reading=(), reference=()):
        super().__init__(min_dist, median_factor, len(reading), len(reference))
        for arr, fl in ((self.reading, reading), (self.reference, reference)):
            for k, (kind, dim, dist) in enumerate(fl):
                arr[k] = DataFilter(kind, dim, dist)


def _compile(out_dir):
    out = os.path.join(out_dir, "libicp_filters_ref.so")
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
        _lib.orc_icp_filtered.restype = ctypes.c_int
        _lib.orc_data_filters.restype = ctypes.c_int
    return _lib


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def data_filters(pts, filters):
    """The data-filter chain [(kind, dim, dist), ...] on pts [N,2] -> survivors float32 [M,2] in input order."""
    lib = _load()
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    fl = IcpFilters(reading=filters)
    out = np.empty_like(pts)
    m = lib.orc_data_filters(fl.reading, len(filters), _fp(pts), len(pts), _fp(out))
    return out[:m].copy()


def icp(src, tgt, guess=None, params=None, filters=None):
    """oracle.icp with the filter block (None: no filter) -> dict(message, T, iterations, inliers, status)."""
    lib = _load()
    src = np.ascontiguousarray(src, np.float32).reshape(-1, 2)
    tgt = np.ascontiguousarray(tgt, np.float32).reshape(-1, 2)
    g = np.eye(3, dtype=np.float32) if guess is None else np.ascontiguousarray(guess, np.float32)
    prm = params or IcpParams()
    fl = filters or IcpFilters()
    T = np.empty((3, 3), np.float32)
    it, inl = ctypes.c_int(0), ctypes.c_int(0)
    st = lib.orc_icp_filtered(_fp(src), len(src), _fp(tgt), len(tgt), _fp(g), ctypes.byref(prm), ctypes.byref(fl),
                              _fp(T), ctypes.byref(it), ctypes.byref(inl))
    return dict(message=ICP_MESSAGES[st], status=st, T=T if st == 0 else g.copy(), iterations=it.value,
                inliers=inl.value)
