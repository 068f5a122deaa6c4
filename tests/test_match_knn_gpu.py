"""GPU: k-nearest-neighbour matching (`pcl.match_knn`, `ops.match` with knn, sfe_match_knn_*) equals the brute-force
oracle (oracle/knn_ref.c orc_match_knn) bit for bit -- ids and squared distances of every slot -- in both launch
classes: references that fit one CTA next to the per-thread lists, and map grids in global memory above that."""
import functools

import numpy as np
import pytest
import torch

from oracle import knn_ref
from sonar_slam_b200 import ops, synth
from sonar_slam_b200.bruce_slam import pcl

pytestmark = pytest.mark.gpu


def _check(ref, pts, knn, max_dist):
    ids, d = pcl.match_knn(ref, pts, knn, max_dist)
    wi, wd = knn_ref.match_knn(ref, pts, knn, max_dist)
    assert ids.shape == (knn, len(pts)) and ids.dtype == np.int32 and d.dtype == np.float32
    assert np.array_equal(ids, wi), (knn, max_dist, np.argwhere(ids != wi)[:5])
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32)), (knn, max_dist)
    return ids, d


def _clouds(kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        ref = rng.uniform(0, 50, (5000, 2))
    elif kind == "lattice":       # equal distances everywhere: the lower index decides
        g = np.arange(60, dtype=np.float64) * 0.5
        ref = np.stack(np.meshgrid(g, g), -1).reshape(-1, 2)[rng.permutation(3600)]
    else:                         # every point two or three times
        base = rng.uniform(0, 30, (1500, 2))
        ref = np.concatenate([base, base[::-1], base[:400]])
    ref = ref.astype(np.float32)
    pts = np.concatenate([ref[rng.integers(len(ref), size=600)] + rng.normal(0, 0.2, (600, 2)),
                          ref[rng.integers(len(ref), size=200)],                          # exact hits
                          rng.uniform(ref.min(0) - 5, ref.max(0) + 5, (200, 2))]).astype(np.float32)
    return ref, pts


@pytest.mark.parametrize("kind", ["random", "lattice", "duplicates"])
@pytest.mark.parametrize("knn", [2, 3, 5, 16])
def test_equals_oracle(gpu_ctx, kind, knn):
    ref, pts = _clouds(kind, knn)
    for max_dist in (0.3, 1.0, np.inf):
        ids, _ = _check(ref, pts, knn, max_dist)
        if max_dist == 0.3:
            assert (ids[-1] == -1).any() and (ids[0] >= 0).any()                   # some slots left empty


def test_edge_cases(gpu_ctx):
    rng = np.random.default_rng(3)
    ref = rng.uniform(0, 10, (300, 2)).astype(np.float32)
    pts = np.concatenate([rng.uniform(-1, 11, (100, 2)), [[np.nan, 2.0], [3.0, np.nan], [np.nan, np.nan]],
                          [[1e30, 0.0], [-1e30, 1e30]]]).astype(np.float32)
    for knn in (2, 16):
        for max_dist in (0.0, 0.5, np.inf, np.nan):
            ids, _ = _check(ref, pts, knn, max_dist)
            assert (ids[:, 100:103] == -1).all()                                     # NaN queries: unmatched
        _check(ref, ref[::3], knn, 0.0)                                              # max_dist 0: the point itself
        _check(ref[:5], pts, knn, np.inf)                                            # knn above the reference size
        _check(ref[:1], pts, knn, 3.0)
        ids, d = _check(np.zeros((0, 2), np.float32), pts, knn, 1.0)                 # empty reference
        assert (ids == -1).all() and np.isinf(d).all()
        ids, d = pcl.match_knn(ref, np.zeros((0, 2), np.float32), knn, 1.0)              # empty query
        assert ids.shape == (knn, 0) and d.shape == (knn, 0)
    for bad, exc in ((0, ValueError), (-1, ValueError), (17, NotImplementedError)):
        with pytest.raises(exc):
            pcl.match_knn(ref, pts, bad, 1.0)


def test_row_zero_is_the_nearest_neighbour_and_rows_are_prefixes(gpu_ctx):
    ref, pts = _clouds("lattice", 9)
    for max_dist in (0.4, 2.0, np.inf):
        one = pcl.match(ref, pts, 1, max_dist)
        full = pcl.match_knn(ref, pts, 16, max_dist)
        assert np.array_equal(full[0][:1], one[0]) and np.array_equal(full[1][:1].view(np.uint32), one[1].view(np.uint32))
        for k in (2, 3, 7, 15):
            part = pcl.match_knn(ref, pts, k, max_dist)
            assert np.array_equal(part[0], full[0][:k]) and np.array_equal(part[1], full[1][:k])


def _cta_limit(knn):
    """Largest reference match_knn_kernel lays out: match_kernel's layout (8 B per point, a cell table of 1.5 entries per
    point, at most 16 384, +16 B), rounded to 16 B, then 6 B per slot of 512 per-thread lists, next to 672 B of static
    shared memory (icp.cu, match_knn_run)."""
    room = torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 672
    lo, hi = 0, 65535
    while lo < hi:
        mid = (lo + hi + 1) // 2
        mc = min(max(mid + mid // 2, 256), 16384)
        need = ((8 * mid + 4 * ((mc + 2) // 2 + 1) + 16 + 15) & ~15) + 512 * knn * 6
        lo, hi = (mid, hi) if need <= room else (lo, mid - 1)
    return lo


@functools.lru_cache(maxsize=None)
def _map(n):
    return synth.make_map_cloud(n, seed=21)[0]


@pytest.mark.parametrize("knn", [2, 16])
@pytest.mark.parametrize("delta", [0, 1])
def test_at_the_one_cta_limit_and_one_past(gpu_ctx, knn, delta):
    """At the limit one match_knn_kernel launch; one point past it that launch plus the map class (nine build launches
    and match_knn_map_kernel)."""
    from sonar_slam_b200 import _lib
    ctx = _lib.default_context()
    ref = _map(60000)[: _cta_limit(knn) + delta]
    rng = np.random.default_rng(knn + delta)
    q = (ref[rng.integers(len(ref), size=1500)] + rng.normal(0, 0.3, (1500, 2))).astype(np.float32)
    n0 = ctx.launches
    _check(ref, q, knn, 1.0)
    assert ctx.launches - n0 == (1 if delta == 0 else 11)


@pytest.mark.parametrize("knn", [3, 16])
def test_map_sized_reference(gpu_ctx, knn):
    ref = _map(150000)
    rng = np.random.default_rng(knn)
    q = np.concatenate([ref[rng.integers(len(ref), size=2000)] + rng.normal(0, 0.3, (2000, 2)),
                        rng.uniform(ref.min(0) - 10, ref.max(0) + 10, (500, 2))]).astype(np.float32)
    for max_dist in (0.5, np.inf):
        _check(ref, q, knn, max_dist)


def test_batched_ops_match_mixes_both_classes(gpu_ctx):
    rng = np.random.default_rng(17)
    refs = [_map(60000)[:30000], rng.uniform(0, 20, (400, 2)), np.zeros((0, 2)), _map(60000)[:5000],
            _map(60000), np.float32([[1, 0], [0, 1], [-1, 0], [1, 0]])]
    refs = [np.asarray(r, np.float32) for r in refs]
    ins = [(r[rng.integers(len(r), size=700)] + rng.normal(0, 0.4, (700, 2))) if len(r) else rng.uniform(0, 5, (30, 2))
           for r in refs[:-1]] + [np.float32([[0, 0], [1, 0]])]
    ins = [np.asarray(i, np.float32) for i in ins]
    ins.insert(3, np.zeros((0, 2), np.float32))                                      # an empty query cloud
    refs.insert(3, rng.uniform(0, 5, (50, 2)).astype(np.float32))

    def pack(clouds):
        off = np.zeros(len(clouds) + 1, np.int32)
        off[1:] = np.cumsum([len(c) for c in clouds])
        return torch.from_numpy(np.concatenate(clouds)).cuda(), torch.from_numpy(off).cuda(), off

    rp, ro, _ = pack(refs)
    ip, io, io_h = pack(ins)
    n_ref_max = max(len(r) for r in refs)
    for knn, md in ((5, 0.8), (16, np.inf)):
        out = ops.match(rp, ro, ip, io, n_ref_max, md, knn=knn)
        one = ops.match(rp, ro, ip, io, n_ref_max, md)
        ids, d = out["ids"].cpu().numpy(), out["dists"].cpu().numpy()
        assert ids.shape == (knn, int(io_h[-1]))
        assert np.array_equal(ids[0], one["ids"].cpu().numpy()) and np.array_equal(d[0], one["dists"].cpu().numpy())
        for c in range(len(refs)):
            wi, wd = knn_ref.match_knn(refs[c], ins[c], knn, md)
            s, e = io_h[c], io_h[c + 1]
            assert np.array_equal(ids[:, s:e], wi), (knn, c)
            assert np.array_equal(d[:, s:e].view(np.uint32), wd.view(np.uint32)), (knn, c)
