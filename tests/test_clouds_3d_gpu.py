"""GPU: [N,3] clouds through `pcl.downsample`, `pcl.match`, `pcl.match_knn` and `ops` -- the octree down-sample
(one-CTA kernel and grid-wide path) and the 3-D nearest / k-nearest match (in-CTA and map classes) -- equal to the CPU
oracles (oracle/cloud3_ref.c orc_downsample3 / orc_match_brute3 / orc_match_knn3) index for index and
bit for bit, and a 3-D cloud with z = 0 equal to the 2-D device path."""
import functools

import numpy as np
import pytest
import torch

from oracle import cloud3_ref as c3
from sonar_slam_b200 import ops, synth
from sonar_slam_b200.bruce_slam import pcl

from oracle.cloud3_ref import octree_literal

pytestmark = pytest.mark.gpu

F = np.float32


@functools.lru_cache(maxsize=None)
def _map3(n, seed=1, z_spread=4.0):
    """A whole-map cloud with depth: synth.make_map_cloud's walls, z uniform over z_spread metres."""
    xy = synth.make_map_cloud(n, seed=seed)[0]
    z = np.random.default_rng(seed + 100).uniform(0, z_spread, n)
    return np.c_[xy, z].astype(F)


def _uniform(n, seed, spread=(40.0, 40.0, 10.0)):
    return (np.random.default_rng(seed).uniform(0, 1, (n, 3)) * np.asarray(spread)).astype(F)


def _check_downsample(pts, res):
    keys = np.arange(len(pts), dtype=F)[:, None]
    got, gk = pcl.downsample(pts, keys, res)
    want, widx = c3.downsample3(pts, res)
    assert got.shape == want.shape and got.dtype == F, (len(pts), res)
    assert np.array_equal(gk[:, 0].astype(np.int64), widx), (len(pts), res)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (len(pts), res)
    assert np.array_equal(pcl.downsample(pts, res), want)
    return widx


def test_one_cta_clouds(gpu_ctx):
    lim = ops.downsample_cta_limit(3)
    assert 1000 < lim < ops.downsample_cta_limit(2)  # 24 bytes of shared memory per point instead of 16
    rng = np.random.default_rng(0)
    g = np.arange(10, dtype=F) * F(0.5)
    lattice = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)[rng.permutation(1000)]
    clouds = [(_uniform(3000, 1), 1.0), (_uniform(2048, 2), 0.3), (_uniform(700, 3, (2, 2, 2)), 0.05),
              (lattice, 0.5), (lattice, 1.3),
              (np.c_[np.full(400, 2.0), np.full(400, -1.0), np.linspace(0, 20, 400)].astype(F), 0.4),  # z only
              (np.tile(F([[1.0, 2.0, 3.0]]), (300, 1)), 0.5),                                        # coincident
              (F([[4.0, 5.0, 6.0]]), 0.5), (np.repeat(_uniform(500, 4), 3, axis=0), 2.0)]
    for pts, res in clouds:
        _check_downsample(pts, res)


def test_clouds_around_the_one_cta_limit(gpu_ctx):
    lim = ops.downsample_cta_limit(3)
    for n in (lim - 1, lim, lim + 1, lim + 500):
        for res in (0.5, 3.0):
            _check_downsample(_uniform(n, n), res)


@pytest.mark.parametrize("res", [0.5, 0.13, 7.0])
def test_map_sized_clouds(gpu_ctx, res):
    _check_downsample(_map3(1_000_000), res)


def test_deeper_than_15_levels_is_cut_there(gpu_ctx):
    """Two dense blobs 2^17 resolutions apart (and sparse points between): the oracle's octree is 18 levels deep, the
    device's stops at 15 on both paths -- the literal octree with its nodes at depth 15 made leaves."""
    rng = np.random.default_rng(5)
    for n_sparse in (300, ops.downsample_cta_limit(3) + 2000):
        pts = np.concatenate([rng.uniform(0, 6, (100, 3)), rng.uniform(0, 400, (n_sparse, 3)),
                              rng.uniform(0, 6, (100, 3)) + 2.0 ** 17]).astype(F)
        keys = np.arange(len(pts), dtype=F)[:, None]
        got, gk = pcl.downsample(pts, keys, 1.0)
        want = octree_literal(pts, 1.0, max_depth=15)
        assert np.array_equal(gk[:, 0].astype(np.int64), want) and np.array_equal(got, pts[want])
        assert len(want) < len(c3.downsample3(pts, 1.0)[1])  # the leaves below level 15 are merged


def _pack(clouds, dev="cuda"):
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    pts = np.concatenate(clouds).astype(F)
    return torch.from_numpy(pts).to(dev), torch.from_numpy(off).to(dev), off


def test_packed_batch_mixing_both_classes(gpu_ctx):
    lim = ops.downsample_cta_limit(3)
    clouds = [_uniform(500, 10), _map3(120_000, seed=2), _uniform(lim, 11), np.zeros((0, 3), F), _uniform(1, 12),
              _uniform(lim + 1, 13), _uniform(3000, 14)]
    pts, off, off_h = _pack(clouds)
    for res in (0.4, 2.0):
        out = ops.downsample(pts, off, max(len(c) for c in clouds), res)
        torch.cuda.synchronize()
        cnt, idx, got = out["count"].cpu().numpy(), out["idx"].cpu().numpy(), out["pts"].cpu().numpy()
        for c, cl in enumerate(clouds):
            want, widx = c3.downsample3(cl, res)
            assert cnt[c] == len(widx), (c, res)
            a = off_h[c]
            assert np.array_equal(idx[a:a + cnt[c]], widx) and np.array_equal(got[a:a + cnt[c]], want), (c, res)


def test_z_zero_equals_the_2d_device_path(gpu_ctx):
    lim2 = ops.downsample_cta_limit(2)
    for xy in (synth.make_map_cloud(3000, seed=3)[0], synth.make_map_cloud(lim2 + 5000, seed=4)[0]):
        flat = np.c_[xy, np.zeros(len(xy))].astype(F)
        for res in (0.5, 2.0):
            d3, d2 = pcl.downsample(flat, res), pcl.downsample(xy, res)
            assert np.array_equal(d3[:, :2], d2) and not d3[:, 2].any()
        q = (xy[::7] + F(0.05)).astype(F)
        q3 = np.c_[q, np.zeros(len(q))].astype(F)
        i3, e3 = pcl.match(flat, q3, 1, 0.3)
        i2, e2 = pcl.match(xy, q, 1, 0.3)
        assert np.array_equal(i3, i2) and np.array_equal(e3.view(np.uint32), e2.view(np.uint32))
        for knn in (2, 5):
            i3, e3 = pcl.match_knn(flat, q3, knn, 0.5)
            i2, e2 = pcl.match_knn(xy, q, knn, 0.5)
            assert np.array_equal(i3, i2) and np.array_equal(e3.view(np.uint32), e2.view(np.uint32))


def _check_match(ref, pts, knn, max_dist):
    ids, d = pcl.match_knn(ref, pts, knn, max_dist) if knn > 1 else pcl.match(ref, pts, 1, max_dist)
    wi, wd = c3.match_knn3(ref, pts, knn, max_dist)
    assert ids.shape == (knn, len(pts)) and ids.dtype == np.int32 and d.dtype == F
    assert np.array_equal(ids, wi), (knn, max_dist, np.argwhere(ids != wi)[:5])
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32)), (knn, max_dist)
    if knn == 1:
        bi, bd = c3.match3(ref, pts, max_dist)
        assert np.array_equal(ids, bi) and np.array_equal(d.view(np.uint32), bd.view(np.uint32))
    return ids


def _queries(ref, rng, n):
    return np.concatenate([ref[rng.integers(len(ref), size=n // 2)] + rng.normal(0, 0.2, (n // 2, 3)),
                           ref[rng.integers(len(ref), size=n // 4)],                                   # exact hits
                           rng.uniform(ref.min(0) - 3, ref.max(0) + 3, (n - n // 2 - n // 4, 3))]).astype(F)


@pytest.mark.parametrize("knn", [1, 2, 5, 16])
def test_match_in_cta_class(gpu_ctx, knn):
    rng = np.random.default_rng(knn)
    base = _uniform(1500, 20 + knn, (20.0, 20.0, 5.0))
    g = np.arange(8, dtype=F) * F(0.5)
    lattice = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    for ref in (_uniform(5000, 30 + knn), np.concatenate([base, base[::-1], base[:300]]), lattice):  # ties
        pts = _queries(ref, rng, 1000)
        for max_dist in (0.3, 1.0, np.inf):
            ids = _check_match(ref, pts, knn, max_dist)
            if max_dist == 0.3 and knn > 1:
                assert (ids[-1] == -1).any() and (ids[0] >= 0).any()  # fewer than knn neighbours
    # points at exactly max_dist: lattice neighbours 0.5 apart, max_dist 0.5 (accepted: dist <= max_dist^2)
    ids = _check_match(lattice, lattice[::5] + F([0.0, 0.0, 0.0]), knn, 0.5)
    assert (ids[min(knn, 2) - 1] >= 0).all()


@pytest.mark.parametrize("knn", [1, 2, 5, 16])
def test_match_map_class(gpu_ctx, knn):
    rng = np.random.default_rng(40 + knn)
    for ref in (_map3(60_000, seed=6), _map3(1_000_000, seed=7)):
        pts = _queries(ref, rng, 1500 if len(ref) < 100_000 else 300)
        for max_dist in (0.2, 2.0):
            _check_match(ref, pts, knn, max_dist)


def test_ops_match_batches_both_classes(gpu_ctx):
    rng = np.random.default_rng(50)
    refs = [_uniform(2000, 51), _map3(60_000, seed=8), np.zeros((0, 3), F), _uniform(1, 52)]
    ins = [_queries(r, rng, 400) if len(r) else _uniform(5, 53) for r in refs]
    rp, ro, _ = _pack(refs)
    ip, io, io_h = _pack(ins)
    for knn in (None, 1, 4):
        out = ops.match(rp, ro, ip, io, max(len(r) for r in refs), 1.0, knn=knn)
        torch.cuda.synchronize()
        ids, d = out["ids"].cpu().numpy(), out["dists"].cpu().numpy()
        k = 1 if knn is None else knn
        ids, d = ids.reshape(k, -1), d.reshape(k, -1)
        for p, (r, q) in enumerate(zip(refs, ins)):
            wi, wd = c3.match_knn3(r, q, k, 1.0)
            a, b = io_h[p], io_h[p + 1]
            assert np.array_equal(ids[:, a:b], wi) and np.array_equal(d[:, a:b].view(np.uint32), wd.view(np.uint32))
