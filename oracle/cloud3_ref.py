"""TEST INFRASTRUCTURE ONLY -- ctypes doorway onto oracle/cloud3_ref.c (down-sample and match on [N,3] clouds).

The library is compiled on first use with the flags of oracle/Makefile's restatements (-O3, -ffp-contract=off: every
float32 product and sum rounded separately) into oracle/_build/libcloud3_ref.so, or into a temporary directory when the
tree is read-only, and rebuilt whenever cloud3_ref.c is newer.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "cloud3_ref.c")
CFLAGS = ["-O3", "-std=c11", "-fPIC", "-ffp-contract=off", "-Wall", "-Wextra", "-shared"]
_lib = None


def _compile(out_dir):
    out = os.path.join(out_dir, "libcloud3_ref.so")
    if os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(_SRC):
        return out
    os.makedirs(out_dir, exist_ok=True)
    tmp = f"{out}.{os.getpid()}.tmp"
    subprocess.run([os.environ.get("CC", "gcc")] + CFLAGS + [_SRC, "-lm", "-o", tmp], check=True)
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
        _lib.orc_downsample3.restype = ctypes.c_int
        _lib.orc_match_brute3.restype = None
        _lib.orc_match_knn3.restype = None
    return _lib


_FP = ctypes.POINTER(ctypes.c_float)
_IP = ctypes.POINTER(ctypes.c_int32)


def _f32x3(a):
    a = np.ascontiguousarray(a, np.float32)
    return a.reshape(-1, 3) if a.size else a.reshape(0, 3)


def downsample3(pts, resolution):
    """pcl.downsample(pts[N,3], resolution): the octree (orc_downsample3) -> (kept points float32, their indices)."""
    lib = _load()
    pts = _f32x3(pts)
    idx = np.empty(len(pts), np.int32)
    m = lib.orc_downsample3(pts.ctypes.data_as(_FP), len(pts), ctypes.c_float(resolution), idx.ctypes.data_as(_IP))
    idx = idx[:m].copy()
    return pts[idx], idx


def match3(ref, pts, max_dist):
    """pcl.match(ref[N,3], pts[M,3], 1, max_dist) by brute force (orc_match_brute3) -> (ids int32 [1,M], squared dists
    float32 [1,M])."""
    lib = _load()
    ref, pts = _f32x3(ref), _f32x3(pts)
    ids = np.empty(len(pts), np.int32)
    d = np.empty(len(pts), np.float32)
    lib.orc_match_brute3(ref.ctypes.data_as(_FP), len(ref), pts.ctypes.data_as(_FP), len(pts), ctypes.c_float(max_dist),
                         ids.ctypes.data_as(_IP), d.ctypes.data_as(_FP))
    return ids[None, :], d[None, :]


def match_knn3(ref, pts, knn, max_dist):
    """pcl.match_knn(ref[N,3], pts[M,3], knn, max_dist) (orc_match_knn3) -> (ids int32 [knn,M], squared dists float32
    [knn,M])."""
    knn = int(knn)
    if knn < 1:
        raise ValueError(f"match_knn3: knn must be at least 1 (got {knn})")
    lib = _load()
    ref, pts = _f32x3(ref), _f32x3(pts)
    ids = np.empty((knn, len(pts)), np.int32)
    d = np.empty((knn, len(pts)), np.float32)
    lib.orc_match_knn3(ref.ctypes.data_as(_FP), len(ref), pts.ctypes.data_as(_FP), len(pts), knn,
                       ctypes.c_float(max_dist), ids.ctypes.data_as(_IP), d.ctypes.data_as(_FP))
    return ids, d
