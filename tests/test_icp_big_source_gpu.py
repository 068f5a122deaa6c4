"""GPU: scan matching with sources of any size.  Sources above what the shared-memory layouts hold
(ops.icp_source_limit) take the global-source class -- per-source-point arrays in global memory, every target read
from a map grid -- and are held to the CPU oracles exactly (status, iterations, inliers, every entry of T): at the
class boundary, above 65 535 points, against small and map-sized targets, in 2-D and 3-D, next to the other classes
in one call.  Calls that fit the shared-memory layouts keep their launches."""
import functools

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import icp3_ref as o3
from oracle import icp_filters_ref as fr
from oracle import oracle as orc
from sonar_slam_b200 import _lib, ops, synth
from sonar_slam_b200.bruce_slam import pcl

pytestmark = pytest.mark.gpu
F32 = np.float32
FIXED20 = dict(max_iterations=20, smooth_length=0)
CHECKERS = {"fixed20": FIXED20, "shipped": {}}
# (raw map points, down-sampling resolution): 30 000 (first 30 000 kept) and 243 726 points, as in test_map_icp_gpu
MAPS = {"30k": (400000, 0.1, 30000), "250k": (1600000, 0.05, None)}
FILTERS = dict(min_dist=0.01, median_factor=1.5, reading=[(_lib.MIN_DIST, -1, 1.0)], reference=[(_lib.MAX_DIST, -1, 400.0)])


@functools.lru_cache(maxsize=None)
def _map(name):
    n, res, keep = MAPS[name]
    return orc.downsample(synth.make_map_cloud(n, seed=11)[0], res)[0][:keep]


@functools.lru_cache(maxsize=None)
def _map3(name):
    """The 2-D map over an undulating floor: z = 0.8 sin(x / 9) cos(y / 7), a few centimetres of noise."""
    m = _map(name).astype(np.float64)
    z = 0.8 * np.sin(m[:, 0] / 9.0) * np.cos(m[:, 1] / 7.0) + np.random.default_rng(3).normal(0, 0.03, len(m))
    return np.c_[m, z].astype(F32)


def _se2(x, y, t):
    c, s = np.cos(t), np.sin(t)
    return np.array([[c, -s, x], [s, c, y], [0, 0, 1]], F32)


def _source(tgt, n, seed):
    """n points of tgt (with repeats when n > len(tgt)), 2 cm of noise, moved into a frame at a known rigid transform
    T about the cloud's centre (source = T^-1 tgt).  Returns (source, T)."""
    rng = np.random.default_rng(seed)
    dim = tgt.shape[1]
    pts = tgt[rng.permutation(len(tgt))[:n] if n <= len(tgt) else rng.integers(len(tgt), size=n)].astype(np.float64)
    pts += rng.normal(0, 0.02, pts.shape)
    c = tgt.mean(0).astype(np.float64)
    if dim == 2:
        T = _se2(c[0] + rng.normal(0, 2), c[1] + rng.normal(0, 2), rng.uniform(-np.pi, np.pi)).astype(np.float64)
    else:
        T = synth.se3(c + rng.normal(0, 2, 3), np.array([0.1, -0.2, 1.0]), rng.uniform(-np.pi, np.pi))
    R, t = T[:dim, :dim], T[:dim, dim]
    return ((pts - t) @ R).astype(F32), T.astype(F32)


def _guesses(T, k, seed):
    """k guesses near T: a few decimetres and a few hundredths of a radian off."""
    rng = np.random.default_rng(seed)
    dim = T.shape[0] - 1
    out = []
    for _ in range(k):
        if dim == 2:
            D = _se2(rng.normal(0, 0.3), rng.normal(0, 0.3), rng.normal(0, 0.03))
        else:
            D = synth.se3(rng.normal(0, 0.3, 3), rng.normal(size=3), rng.normal(0, 0.03)).astype(F32)
        out.append((D.astype(np.float64) @ T.astype(np.float64)).astype(F32))
    return out


def _icp(filters=None, **kw):
    icp = pcl.ICP()
    icp.params = _lib.IcpConfig(filters=None if filters is None else _lib.IcpFilters(**filters), **kw)
    return icp


def _want(src, tgt, guess, kw, filters=None):
    if src.shape[1] == 3:
        return o3.icp3(src, tgt, guess, orc.IcpParams(**kw))
    if filters is not None:
        return fr.icp(src, tgt, guess, orc.IcpParams(**kw), fr.IcpFilters(**filters))
    return orc.icp(src, tgt, guess, orc.IcpParams(**kw))


def _assert_same(res, k, want, what):
    got = (int(res["status"][k]), int(res["iterations"][k]), int(res["inliers"][k]))
    assert got == (want["status"], want["iterations"], want["inliers"]), (what, got, want)
    assert np.asarray(res["T"][k], F32).tobytes() == np.asarray(want["T"], F32).tobytes(), (what, res["T"][k], want["T"])


def _check_batch(src, tgt, guesses, kw, what, filters=None):
    """compute_batch on one pair against the oracle, guess by guess; returns the device results"""
    res = _icp(filters, **kw).compute_batch(src, tgt, guesses)
    for k, g in enumerate(guesses):
        _assert_same(res, k, _want(src, tgt, g, kw, filters), f"{what} guess {k}")
    return res


def _limit(dim, kw=None, filters=None):
    lim = ops.icp_source_limit(dim, _lib.IcpParams(**(kw or {})),
                               filters=None if filters is None else _lib.IcpFilters(**filters))
    assert 1536 < lim < 65535
    return lim


# ------------------------------------------------------------------ 1, 2: the class boundary
BOUNDARY_2D = {"point": (dict(FIXED20), None), "plane": (dict(minimizer=1, normals_knn=5, **FIXED20), None),
               "filters": (dict(FIXED20), FILTERS)}


@pytest.mark.parametrize("name", list(BOUNDARY_2D))
def test_boundary_2d(gpu_ctx, name):
    """Sources of limit points run in the map class, limit + 1 in the global-source class: one launch more (point to
    point: the in-CTA launch, empty here, map_build's nine and the map class, then the global-source launch)."""
    kw, filters = BOUNDARY_2D[name]
    tgt = _map("30k")
    lim = _limit(2, kw, filters)
    ctx = _lib.default_context()
    counts = []
    for delta in (0, 1):
        src, T = _source(tgt, lim + delta, 40 + delta)
        n0 = ctx.launches
        res = _check_batch(src, tgt, _guesses(T, 2, 41), kw, f"{name} {lim + delta}", filters)
        counts.append(ctx.launches - n0)
        assert (res["status"] == 0).all()
    assert counts[1] == counts[0] + 1
    if name == "point":
        assert counts[0] == 11


def test_boundary_3d(gpu_ctx):
    """The same call at the limit (shared-memory classes) and one point past it (one launch more: the global source)."""
    tgt = _map3("30k")
    lim = _limit(3)
    assert lim > _limit(2)  # 20 bytes of shared memory per source point instead of 27
    ctx = _lib.default_context()
    counts = []
    for delta in (0, 1):
        src, T = _source(tgt, lim + delta, 50 + delta)
        gs = _guesses(T, 2, 51)
        n0 = ctx.launches
        res = _icp(**FIXED20).compute_batch(src, tgt, gs)
        counts.append(ctx.launches - n0)
        for k, g in enumerate(gs):
            _assert_same(res, k, _want(src, tgt, g, FIXED20), f"3-D {lim + delta} guess {k}")
        assert (res["status"] == 0).all()
    assert counts[1] == counts[0] + 1


# ------------------------------------------------------------------ 3: above 65 535 points
@pytest.mark.parametrize("checkers", list(CHECKERS))
@pytest.mark.parametrize("target", ["small", "250k"])
@pytest.mark.parametrize("n", [70000, 150000])
@pytest.mark.parametrize("dim", [2, 3])
def test_sources_above_16_bit_indices(gpu_ctx, dim, n, target, checkers):
    kw = CHECKERS[checkers]
    if target == "small":
        if dim == 2:
            src, tgt, T = synth.make_icp_pair(60 + n // 1000, n_source=n, n_target=3000)
        else:
            src, tgt, T = synth.make_icp_pair3(60 + n // 1000, n_source=n, n_target=3000)
        assert len(tgt) < 5000
        T = T.astype(F32)
        guesses = [np.eye(dim + 1, dtype=F32), T]
    else:
        tgt = _map(target) if dim == 2 else _map3(target)
        src, T = _source(tgt, n, n // 1000)
        guesses = _guesses(T, 2, n // 1000)
    assert len(src) == n > 65535
    res = _check_batch(src, tgt, guesses, kw, f"{dim}-D {n} x {len(tgt)}")
    assert (res["status"] == 0).any()


# ------------------------------------------------------------------ 4: the three classes in one call
@pytest.mark.parametrize("dim", [2, 3])
def test_mixed_call(gpu_ctx, dim):
    """In-CTA, map-target and global-source problems in one compute_pairs call: each equals the oracle, and equals the
    same problem solved alone."""
    lim = _limit(dim)
    big = _map("250k") if dim == 2 else _map3("250k")
    make = synth.make_icp_pair if dim == 2 else synth.make_icp_pair3
    pairs = []
    for c in range(3):  # in-CTA (targets that fit one CTA next to limit-point sources)
        s, t, T = make(700 + c, n_source=800, n_target=800)
        pairs.append((s, t, [np.eye(dim + 1, dtype=F32), T.astype(F32)]))
    s, T = _source(big, 1500, 5)  # map target
    pairs.append((s, big, _guesses(T, 2, 5)))
    s, t, T = make(710, n_source=lim + 5000, n_target=3000)  # global source, small target
    pairs.append((s, t, [T.astype(F32)]))
    s, T = _source(big, 80000, 6)  # global source, map target
    pairs.append((s, big, _guesses(T, 2, 6)))
    order = np.random.default_rng(dim).permutation(len(pairs))
    pairs = [pairs[i] for i in order]
    icp = _icp()
    out = icp.compute_pairs([p[0] for p in pairs], [p[1] for p in pairs], [p[2] for p in pairs])
    for (s, t, gs), r in zip(pairs, out):
        alone = icp.compute_batch(s, t, gs)
        for k, g in enumerate(gs):
            _assert_same(r, k, _want(s, t, g, {}), f"{dim}-D mixed {len(s)} x {len(t)}")
        for key in ("T", "iterations", "inliers", "status"):
            assert np.array_equal(r[key], alone[key]), key


# ------------------------------------------------------------------ 5: float64 accumulation
def _f64_icp(src, tgt, guess, iters):
    """float64 numpy + cKDTree arm of test_icp_parity_gpu: NN within 10 m, MaxDist 3 m, Trimmed 0.8, 2-D rigid fit."""
    src, tgt = src.astype(np.float64), tgt.astype(np.float64)
    tree = cKDTree(tgt)
    T = np.array(guess, np.float64)
    for _ in range(iters):
        p = src @ T[:2, :2].T + T[:2, 2]
        d, j = tree.query(p, distance_upper_bound=10.0)
        fin = np.isfinite(d)
        d2 = d ** 2
        lim = np.sort(d2[fin])[int(np.float32(fin.sum()) * np.float32(0.8))]
        keep = fin & (d2 <= 9.0) & (d2 <= lim)
        a, b = p[keep], tgt[j[keep]]
        ma, mb = a.mean(0), b.mean(0)
        H = (b - mb).T @ (a - ma)
        th = np.arctan2(H[1, 0] - H[0, 1], H[0, 0] + H[1, 1])
        R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
        D = np.eye(3)
        D[:2, :2], D[:2, 2] = R, mb - R @ ma
        T = D @ T
    return T


def _pose(T):
    T = np.asarray(T, np.float64)
    return np.array([T[0, 2], T[1, 2], np.arctan2(T[1, 0], T[0, 0])])


def test_float64_mode_on_a_big_source(gpu_ctx):
    tgt = _map("250k")
    src, T = _source(tgt, 70000, 8)
    gs = _guesses(T, 2, 8)
    res = _icp(flags=2, **FIXED20).compute_batch(src, tgt, gs)
    assert (res["status"] == 0).all() and (res["iterations"] == 20).all()
    for k, g in enumerate(gs):
        dev = np.abs(_pose(res["T"][k]) - _pose(_f64_icp(src, tgt, g, 20)))
        assert dev.max() < 5e-3, dev


# ------------------------------------------------------------------ 6: guards
def _packed(clouds, dim):
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    pts = np.concatenate([np.asarray(c, F32).reshape(-1, dim) for c in clouds])
    return torch.from_numpy(np.ascontiguousarray(pts)).cuda(), torch.from_numpy(off).cuda()


def _ops_icp(srcs, tgts, guesses, ns_max=None, **kw):
    dim = srcs[0].shape[1]
    sp, so = _packed(srcs, dim)
    tp, to = _packed(tgts, dim)
    g = torch.from_numpy(np.stack(guesses).astype(F32)).cuda()
    out = ops.icp(sp, so, tp, to, g, ns_max or max(map(len, srcs)), max(map(len, tgts)), _lib.IcpParams(**kw))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("dim", [2, 3])
def test_too_large_and_empty_target(gpu_ctx, dim):
    lim = _limit(dim)
    tgt = _map("30k") if dim == 2 else _map3("30k")
    src, T = _source(tgt, 70000, 9)
    small, _ = _source(tgt, 2000, 10)
    g = _guesses(T, 1, 9)[0]
    # a source above the ns_max the call declares is reported too large, whatever class the call runs
    r = _ops_icp([src, small], [tgt, tgt], [g, g], ns_max=lim + 1000, **FIXED20)
    assert r["status"][0] == 8 and r["iterations"][0] == 0 and np.array_equal(r["T"][0], g)
    _assert_same(r, 1, _want(small, tgt, g, FIXED20), "small source next to a too-large one")
    # an empty target next to a big source: SFE_ICP_EMPTY_REF, next to other targets and as the call's only target
    empty = np.zeros((0, dim), F32)
    r = _ops_icp([src, src], [empty, tgt], [g, g], **FIXED20)
    assert r["status"][0] == 6 and np.array_equal(r["T"][0], g)
    _assert_same(r, 1, _want(src, tgt, g, FIXED20), "big source next to an empty target")
    assert gpu_ctx.lib.sfe_icp_status_message(6).decode() == "reference cloud is empty"
    with pytest.raises(RuntimeError, match="reference cloud is empty"):
        _icp().compute(src, empty, np.eye(dim + 1, dtype=F32))


@pytest.mark.parametrize("dim", [2, 3])
def test_source_too_large_for_one_slice(gpu_ctx, dim):
    """A source whose one workspace slice exceeds 512 MiB fails with SFE_ERR_UNSUPPORTED and a message, before any
    launch; the context keeps working."""
    n = (512 << 20) // (29 if dim == 2 else 20) + 1000
    src = np.zeros((n, dim), F32)
    src[:, 0] = np.arange(n, dtype=F32) * F32(1e-3)
    tgt = _map("30k") if dim == 2 else _map3("30k")
    ctx = ops.context(0)
    n0 = ctx.launches
    with pytest.raises(_lib.SonarFEError, match=r"code -4\).*global workspace per CTA"):
        _ops_icp([src], [tgt], [np.eye(dim + 1, dtype=F32)])
    assert ctx.launches == n0
    small, T = _source(tgt, 2000, 12)
    g = _guesses(T, 1, 12)[0]
    _assert_same(_ops_icp([small], [tgt], [g], **FIXED20), 0, _want(small, tgt, g, FIXED20), "after the refusal")


# ------------------------------------------------------------------ 7: calls the shared-memory layouts hold
@pytest.mark.parametrize("dim", [2, 3])
def test_calls_that_fit_keep_their_launches(gpu_ctx, dim):
    """One launch for a call whose targets fit one CTA next to its sources -- also for sources a little above the
    source limit next to small targets, which the in-CTA layout still holds -- and no global-source launch for a source
    at the limit against a map target."""
    ctx = _lib.default_context()
    lim = _limit(dim)
    make = synth.make_icp_pair if dim == 2 else synth.make_icp_pair3
    for ns, nt in ((800, 3000), (lim, 300), (lim + 50, 300)):
        s, t, T = make(90, n_source=ns, n_target=nt)
        s, t = s[:ns], t[:nt]
        assert ops.icp_cta_limit(dim, len(s)) >= len(t)
        n0 = ctx.launches
        res = _icp(**FIXED20).compute_batch(s, t, [T.astype(F32)])
        assert ctx.launches - n0 == 1, (ns, nt)
        _assert_same(res, 0, _want(s, t, T.astype(F32), FIXED20), f"{dim}-D {ns} x {nt}")
