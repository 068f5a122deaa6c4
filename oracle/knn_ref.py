"""TEST INFRASTRUCTURE ONLY -- ctypes doorway onto oracle/knn_ref.c (brute-force k-nearest-neighbour match).

The library is compiled on first use with the flags of oracle/Makefile's restatements (-O3, -ffp-contract=off: every
float32 product and sum rounded separately) into oracle/_build/libknn_ref.so, or into a temporary directory when the
tree is read-only, and rebuilt whenever knn_ref.c is newer.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "knn_ref.c")
CFLAGS = ["-O3", "-std=c11", "-fPIC", "-ffp-contract=off", "-Wall", "-Wextra", "-shared"]
_lib = None


def _compile(out_dir):
    out = os.path.join(out_dir, "libknn_ref.so")
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
        _lib.orc_match_knn.restype = None
    return _lib


def match_knn(ref, pts, knn, max_dist):
    """pcl.match(ref, pts, knn, max_dist) -> (ids int32 [knn,N], squared dists float32 [knn,N]) (orc_match_knn)."""
    knn = int(knn)
    if knn < 1:
        raise ValueError(f"match_knn: knn must be at least 1 (got {knn})")
    lib = _load()
    ref = np.ascontiguousarray(ref, np.float32).reshape(-1, 2)
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    ids = np.empty((knn, len(pts)), np.int32)
    d = np.empty((knn, len(pts)), np.float32)
    fp = ctypes.POINTER(ctypes.c_float)
    lib.orc_match_knn(ref.ctypes.data_as(fp), len(ref), pts.ctypes.data_as(fp), len(pts), knn,
                      ctypes.c_float(max_dist), ids.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                      d.ctypes.data_as(fp))
    return ids, d
