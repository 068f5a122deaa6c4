"""TEST INFRASTRUCTURE ONLY -- ctypes doorway onto oracle/icp3_ref.c (ICP on [N,3] clouds with 4x4 guesses, and its
3x3 SVD, quaternion and nearest-neighbour pieces).

The library is compiled on first use with the flags of oracle/Makefile's restatements (-O3, -ffp-contract=off: every
float32 product and sum rounded separately) into oracle/_build/libicp3_ref.so, or into a temporary directory when the
tree is read-only, and rebuilt whenever icp3_ref.c is newer.  The calls release the GIL (ctypes), so problems can be
solved on several host threads (icp3_many).
"""
import ctypes
import os
import subprocess
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .oracle import ICP_MESSAGES, IcpParams

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "icp3_ref.c")
CFLAGS = ["-O3", "-std=c11", "-fPIC", "-ffp-contract=off", "-Wall", "-Wextra", "-shared"]
_lib = None
_FP = ctypes.POINTER(ctypes.c_float)
_IP = ctypes.POINTER(ctypes.c_int32)


def _compile(out_dir):
    out = os.path.join(out_dir, "libicp3_ref.so")
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
        lib = ctypes.CDLL(path)
        for name, res in (("orc_icp3", ctypes.c_int), ("orc_svd3", ctypes.c_int), ("orc_rot3", ctypes.c_int),
                          ("orc_det3", ctypes.c_float), ("orc_angular_distance3", ctypes.c_float),
                          ("orc_quat3", None), ("orc_nn3_match", None)):
            getattr(lib, name).restype = res
        _lib = lib
    return _lib


def _f32(a, shape):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(shape))


def _pts3(a):
    a = np.ascontiguousarray(a, np.float32)
    return a.reshape(-1, 3) if a.size else a.reshape(0, 3)


def svd3(M):
    """Eigen's JacobiSVD of the 3x3 M, restated -> (U, S, V, sweeps); sweeps -1: non-finite M (U = V = I, S NaN)."""
    lib = _load()
    M = _f32(M, (3, 3))
    U, V, S = np.empty((3, 3), np.float32), np.empty((3, 3), np.float32), np.empty(3, np.float32)
    n = lib.orc_svd3(M.ctypes.data_as(_FP), U.ctypes.data_as(_FP), S.ctypes.data_as(_FP), V.ctypes.data_as(_FP))
    return U, S, V, n


def rot3(M):
    """R = U V^T of svd3(M) with Sorkine's reflection fix -> (R, fixed); fixed 1: the fix applied, -1: non-finite M."""
    lib = _load()
    M = _f32(M, (3, 3))
    R = np.empty((3, 3), np.float32)
    return R, lib.orc_rot3(M.ctypes.data_as(_FP), R.ctypes.data_as(_FP))


def det3(m):
    """The determinant of a 3x3 (or of a 4x4's top-left 3x3) in the oracle's order."""
    m = np.ascontiguousarray(m, np.float32)
    return float(_load().orc_det3(m.ctypes.data_as(_FP), m.shape[1]))


def quat3(m):
    """Eigen's rotation-matrix -> quaternion conversion of a 3x3 (or a 4x4's top-left 3x3) -> (w, x, y, z) float32."""
    m = np.ascontiguousarray(m, np.float32)
    q = np.empty(4, np.float32)
    _load().orc_quat3(m.ctypes.data_as(_FP), m.shape[1], q.ctypes.data_as(_FP))
    return q


def angular_distance3(a, b):
    """Eigen's angularDistance of the quaternions a, b (w, x, y, z)."""
    a, b = _f32(a, 4), _f32(b, 4)
    return float(_load().orc_angular_distance3(a.ctypes.data_as(_FP), b.ctypes.data_as(_FP)))


def nn3_match(ref, pts, max_dist):
    """The ICP's exact nearest-neighbour search on its own: (ids int32 [M], squared dists float32 [M])."""
    lib = _load()
    ref, pts = _pts3(ref), _pts3(pts)
    ids = np.empty(len(pts), np.int32)
    d = np.empty(len(pts), np.float32)
    lib.orc_nn3_match(ref.ctypes.data_as(_FP), len(ref), pts.ctypes.data_as(_FP), len(pts), ctypes.c_float(max_dist),
                      ids.ctypes.data_as(_IP), d.ctypes.data_as(_FP))
    return ids, d


def icp3(src, tgt, guess=None, params=None):
    """pcl.ICP().compute(src[N,3], tgt[M,3], guess 4x4) -> dict(message, T float32 4x4, iterations, inliers, status)."""
    lib = _load()
    src, tgt = _pts3(src), _pts3(tgt)
    g = np.eye(4, dtype=np.float32) if guess is None else _f32(guess, (4, 4))
    prm = params or IcpParams()
    T = np.empty((4, 4), np.float32)
    it, inl = ctypes.c_int(0), ctypes.c_int(0)
    st = lib.orc_icp3(src.ctypes.data_as(_FP), len(src), tgt.ctypes.data_as(_FP), len(tgt), g.ctypes.data_as(_FP),
                      ctypes.byref(prm), T.ctypes.data_as(_FP), ctypes.byref(it), ctypes.byref(inl))
    return dict(message=ICP_MESSAGES[st], status=st, T=T if st == 0 else g.copy(), iterations=it.value,
                inliers=inl.value)


def icp3_many(problems, params=None, threads=None):
    """icp3 over [(src, tgt, guess), ...] on `threads` host threads (default: every CPU) -> list of icp3's dicts."""
    _load()
    with ThreadPoolExecutor(max_workers=threads or os.cpu_count()) as ex:
        return list(ex.map(lambda p: icp3(p[0], p[1], p[2], params), problems))
