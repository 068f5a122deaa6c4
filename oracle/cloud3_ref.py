"""TEST INFRASTRUCTURE ONLY -- ctypes doorway onto oracle/cloud3_ref.c (down-sample and match on [N,3] clouds).
octree_literal: a second, literal statement of the 3-D down-sample in Python float32 scalars, with an optional depth cut.

The library is compiled on first use with the flags of oracle/Makefile's restatements (-O3, -ffp-contract=off: every
float32 product and sum rounded separately) into oracle/_build/libcloud3_ref.so, or into a temporary directory when the
tree is read-only, and rebuilt whenever cloud3_ref.c is newer.
"""
import ctypes
import os
import subprocess
import sys
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


_F = np.float32


def octree_literal(pts, resolution, max_depth=None):
    """A second statement of the 3-D down-sample: the recursive octree of libpointmatcher's Octree_<T,3>, built node by
    node with float32 scalars (centre = min + extent * 0.5 per axis, half-size = the largest half-extent, split while
    2 * radius > resolution and more than one point, children by x > cx | y > cy << 1 | z > cz << 2 in index order,
    medoid = first minimum of the sequential float32 sum of sqrt((dx*dx + dy*dy) + dz*dz)).  max_depth: nodes at that
    depth become leaves (the device's cut at 15 levels).  Returns the kept indices in output order."""
    pts = np.asarray(pts, _F)
    n = len(pts)
    if n == 0:
        return np.zeros(0, np.int64)
    res = _F(resolution)
    mn, mx = pts.min(0), pts.max(0)
    ext = [_F(mx[d] - mn[d]) for d in range(3)]
    ctr = [_F(mn[d] + _F(ext[d] * _F(0.5))) for d in range(3)]
    radius = max(_F(e * _F(0.5)) for e in ext)
    out = []

    def leaf(idx):
        best, med = _F(np.finfo(_F).max), 0
        for a in idx:
            acc = _F(0)
            for b in idx:
                dx, dy, dz = (_F(pts[a, d] - pts[b, d]) for d in range(3))
                acc = _F(acc + np.sqrt(_F(_F(_F(dx * dx) + _F(dy * dy)) + _F(dz * dz))))
            if acc < best:
                best, med = acc, a
        out.append(med)

    def build(idx, c, r, depth):
        if not idx:
            return
        if float(r) * 2.0 <= float(res) or len(idx) <= 1 or (max_depth is not None and depth >= max_depth):
            leaf(idx)
            return
        kids = [[] for _ in range(8)]
        for i in idx:
            kids[int(pts[i, 0] > c[0]) | int(pts[i, 1] > c[1]) << 1 | int(pts[i, 2] > c[2]) << 2].append(i)
        hr = _F(r * _F(0.5))
        for k in range(8):
            nc = [_F(c[d] + (hr if (k >> d) & 1 else -hr)) for d in range(3)]
            build(kids[k], nc, hr, depth + 1)

    sys.setrecursionlimit(max(sys.getrecursionlimit(), 10000))
    build(list(range(n)), ctr, radius, 0)
    return np.asarray(out, np.int64)
