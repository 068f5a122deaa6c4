"""GPU: the launches of one ICP call partition its problems.  With S the source limit (ops.icp_source_limit) and L
the in-CTA target limit next to S-point sources (ops.icp_cta_limit), a call takes every problem in exactly one launch:
in-CTA {ns <= S, nt <= L}, map {ns <= S, nt > L}, global-source {ns > S} -- or, with no global-source launch, in-CTA
{nt <= L} and map {nt > L}.  Sources small, at S, at S + 1 and above the declared ns_max meet targets that are empty,
at L, at L + 1 and map-sized, in one call per setting; every result equals the CPU oracle and the same problem solved
alone, and the call makes the launches the rule gives."""
import functools

import numpy as np
import pytest
import torch

from oracle import icp3_ref as o3
from oracle import icp_filters_ref as fr
from oracle import oracle as orc
from sonar_slam_b200 import _lib, ops, synth

pytestmark = pytest.mark.gpu
F32 = np.float32
FIXED20 = dict(max_iterations=20, smooth_length=0)
FILTERS = dict(min_dist=0.01, median_factor=1.5, reading=[(_lib.MIN_DIST, -1, 1.0)], reference=[(_lib.MAX_DIST, -1, 400.0)])
# (dim, ICP settings, filters)
SETTINGS = {"2d-point": (2, FIXED20, None), "2d-plane": (2, dict(minimizer=1, normals_knn=5, **FIXED20), None),
            "2d-filters": (2, FIXED20, FILTERS), "3d-point": (3, FIXED20, None)}
TOO_LARGE, EMPTY_REF = 8, 6


@functools.lru_cache(maxsize=None)
def _map(dim):
    """30 000 points of a down-sampled map; in 3-D over an undulating floor (as test_icp_big_source_gpu)"""
    m = orc.downsample(synth.make_map_cloud(400000, seed=11)[0], 0.1)[0][:30000]
    if dim == 2:
        return m
    m = m.astype(np.float64)
    z = 0.8 * np.sin(m[:, 0] / 9.0) * np.cos(m[:, 1] / 7.0) + np.random.default_rng(3).normal(0, 0.03, len(m))
    return np.c_[m, z].astype(F32)


def _near(cloud, n):
    """the n points of cloud nearest (in x, y) to its centre"""
    d = np.linalg.norm(cloud[:, :2] - cloud[:, :2].mean(0), axis=1)
    return cloud[np.argsort(d, kind="stable")[:n]]


def _motion(dim, seed):
    rng = np.random.default_rng(seed)
    if dim == 2:
        c, s = np.cos(0.2), np.sin(0.2)
        T = np.array([[c, -s, 1.5], [s, c, -0.8], [0, 0, 1]])
    else:
        T = synth.se3(np.array([1.5, -0.8, 0.2]), np.array([0.1, -0.2, 1.0]), 0.2)
    D = np.eye(dim + 1)
    D[:dim, dim] = rng.normal(0, 0.2, dim)
    return T.astype(F32), (D @ T).astype(F32)


def _source(dim, n, seed):
    """n map points around the centre, 2 cm of noise, moved by T^-1; returns (source, guess near T)"""
    rng = np.random.default_rng(seed)
    T, guess = _motion(dim, seed)
    pts = _near(_map(dim), n).astype(np.float64) + rng.normal(0, 0.02, (n, dim))
    R, t = T[:dim, :dim].astype(np.float64), T[:dim, dim].astype(np.float64)
    return ((pts - t) @ R).astype(F32), guess


def _packed(clouds, dim):
    """(points, offsets) on the device; one unused row after the last cloud, so that empty clouds alone still pass a
    buffer"""
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    pts = np.concatenate([np.asarray(c, F32).reshape(-1, dim) for c in clouds] + [np.zeros((1, dim), F32)])
    return torch.from_numpy(np.ascontiguousarray(pts)).cuda(), torch.from_numpy(off).cuda()


def _call(srcs, tgts, guesses, ns_max, kw, filters):
    """one ops.icp call on problems (srcs[p], tgts[p], guesses[p]); returns (results, launches)"""
    dim = srcs[0].shape[1]
    sp, so = _packed(srcs, dim)
    tp, to = _packed(tgts, dim)
    g = torch.from_numpy(np.stack(guesses).astype(F32)).cuda()
    ctx = ops.context(0)
    n0 = ctx.launches
    out = ops.icp(sp, so, tp, to, g, ns_max, max(map(len, tgts)), _lib.IcpParams(**kw),
                  filters=None if filters is None else _lib.IcpFilters(**filters))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}, ctx.launches - n0


def _want(src, tgt, guess, ns_max, kw, filters):
    if len(src) > ns_max:
        return dict(status=TOO_LARGE, iterations=0, inliers=0, T=guess)
    if len(tgt) == 0:
        return dict(status=EMPTY_REF, iterations=0, inliers=0, T=guess)
    if src.shape[1] == 3:
        return o3.icp3(src, tgt, guess, orc.IcpParams(**kw))
    if filters is not None:
        return fr.icp(src, tgt, guess, orc.IcpParams(**kw), fr.IcpFilters(**filters))
    return orc.icp(src, tgt, guess, orc.IcpParams(**kw))


def _row(res, k):
    return (int(res["status"][k]), int(res["iterations"][k]), int(res["inliers"][k]),
            np.asarray(res["T"][k], F32).tobytes())


@pytest.mark.parametrize("name", list(SETTINGS))
def test_one_call_partitions_its_problems(gpu_ctx, name):
    dim, kw, filters = SETTINGS[name]
    flt = None if filters is None else _lib.IcpFilters(**filters)
    S = ops.icp_source_limit(dim, _lib.IcpParams(**kw), filters=flt)
    L = ops.icp_cta_limit(dim, S)
    assert 1536 < S < 65535 and 0 < L < 30000
    # (the in-CTA layout of the point-to-point chain without filters: point to plane adds nothing next to sources above
    # 640 points, and the FILT instantiations take the same shared memory)
    tgts = [np.zeros((0, dim), F32), _near(_map(dim), L), _near(_map(dim), L + 1), _map(dim)]
    # the map-sized, small-source problem alone: the in-CTA launch, map_build (and dim 3 the grids' z), the map launch
    small = _source(dim, 700, 1)
    _, n_ref = _call([small[0]], [tgts[3]], [small[1]], 700, kw, filters)
    if name == "2d-point":
        assert n_ref == 11
    cache = {}
    for ns_max, sizes, extra in ((S + 1, (700, S, S + 1, S + 2), 1), (S, (700, S, S + 1), 0)):
        srcs = [_source(dim, n, 10 + n - S) if n != 700 else small for n in sizes]
        probs = [(i, j) for i in range(len(srcs)) for j in range(len(tgts))]
        res, n = _call([srcs[i][0] for i, _ in probs], [tgts[j] for _, j in probs], [srcs[i][1] for i, _ in probs],
                       ns_max, kw, filters)
        # with a global-source launch (ns_max above S) one launch more than the call without it
        assert n == n_ref + extra, (ns_max, n, n_ref)
        for k, (i, j) in enumerate(probs):
            src, guess = srcs[i]
            what = f"{name}: ns_max {ns_max}, source {len(src)} x target {len(tgts[j])}"
            key = (len(src), j, len(src) > ns_max)
            if key not in cache:
                w = _want(src, tgts[j], guess, ns_max, kw, filters)
                cache[key] = (w["status"], w["iterations"], w["inliers"], np.asarray(w["T"], F32).tobytes())
            assert _row(res, k) == cache[key], what
            alone, _ = _call([src], [tgts[j]], [guess], ns_max, kw, filters)
            assert _row(alone, 0) == _row(res, k), what
        assert (res["status"] == 0).any()


@pytest.mark.parametrize("dim", [2, 3])
def test_only_empty_targets_beside_a_global_source(gpu_ctx, dim):
    """A source no shared-memory layout holds next to empty targets only: the in-CTA launch and the global-source launch,
    no map grid, and every problem reports SFE_ICP_EMPTY_REF once."""
    big, g = _source(dim, 20000, 3)  # (more than an in-CTA layout holds next to a one-point target)
    small, g2 = _source(dim, 700, 4)
    empty = np.zeros((0, dim), F32)
    res, n = _call([big, small, big], [empty, empty, empty], [g, g2, g], len(big), FIXED20, None)
    assert n == 2
    assert (res["status"] == EMPTY_REF).all() and (res["iterations"] == 0).all() and (res["inliers"] == 0).all()
    for k, gk in enumerate([g, g2, g]):
        assert np.array_equal(res["T"][k], gk)
