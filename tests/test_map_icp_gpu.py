"""GPU: scan matching and nearest-neighbour matching against map-sized targets -- targets above what one CTA's shared
memory holds, up to a quarter of a million points, run in the map class (map grids in global memory) -- compared
exactly with the CPU oracle (status, iterations, inliers, every entry of T; match ids and squared distances)."""
import functools

import numpy as np
import pytest

from oracle import oracle as orc
from sonar_slam_b200 import synth

pytestmark = pytest.mark.gpu

# (raw map points, down-sampling resolution, points kept): 30 000, 70 916 and 243 726 points
SIZES = {"30k": (400000, 0.1, 30000), "80k": (600000, 0.1, None), "250k": (1600000, 0.05, None)}
FIXED20 = dict(max_iterations=20, smooth_length=0)


@functools.lru_cache(maxsize=None)
def _map(name):
    n, res, keep = SIZES[name]
    return orc.downsample(synth.make_map_cloud(n, seed=11)[0], res)[0][:keep]


def _se2(x, y, t):
    c, s = np.cos(t), np.sin(t)
    return np.array([[c, -s, x], [s, c, y], [0, 0, 1]], np.float32)


def _source(tgt, n, seed):
    """n map points within 30 m of a map point, moved into a frame at a known SE(2) (source = T^-1 map)."""
    rng = np.random.default_rng(seed)
    centre = tgt[rng.integers(len(tgt))]
    near = tgt[np.linalg.norm(tgt - centre, axis=1) < 30.0]
    pts = near[rng.choice(len(near), min(n, len(near)), replace=False)]
    T = _se2(centre[0] + rng.normal(0, 2), centre[1] + rng.normal(0, 2), rng.uniform(-np.pi, np.pi))
    R, t = T[:2, :2].astype(np.float64), T[:2, 2].astype(np.float64)
    src = ((pts - t) @ R).astype(np.float32)  # R^T (p - t), row vectors
    return src, T


def _guesses(T, k, seed):
    rng = np.random.default_rng(seed)
    th = np.arctan2(T[1, 0], T[0, 0])
    return [_se2(T[0, 2] + rng.normal(0, 0.3), T[1, 2] + rng.normal(0, 0.3), th + rng.normal(0, 0.03))
            for _ in range(k)]


def _params(**kw):
    from sonar_slam_b200 import _lib
    return _lib.IcpParams(**kw), orc.IcpParams(**kw)


def _icp(prm):
    from sonar_slam_b200.bruce_slam import pcl
    icp = pcl.ICP()
    icp.params = prm
    return icp


def _assert_oracle(res, k, src, tgt, guess, oprm):
    want = orc.icp(src, tgt, guess, oprm)
    assert int(res["status"][k]) == want["status"]
    assert int(res["iterations"][k]) == want["iterations"] and int(res["inliers"][k]) == want["inliers"]
    assert np.array_equal(res["T"][k], want["T"]), (res["T"][k], want["T"])
    return want


def _cta_limit(ns, plane=False):
    """Largest target icp_kernel lays out next to an ns-point source: icp.cu's icp_cta_smem (8 B per target point, a
    cell table of 1.5 entries per point trimmed down to nt/4 + 256, the source arrays) against the opt-in limit."""
    import torch
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    shared = 5712  # sizeof(IcpShared), rounded up to 16

    def smem(nt, mc):
        order = ns > 1024
        return (shared + 8 * nt + 4 * ((mc + 2) // 2 + 1) + 8 + 8 * ns + 4 * ns + 4 * ns + ns + 4 + 4 * ns
                + (2 * ns if order else 0) + 16 + (16 + 640 * 4 if plane and ns < 640 else 0))

    def fits(nt):
        mc = min(max(nt + nt // 2, 256), 16384)
        while smem(nt, mc) > optin and mc > nt // 4 + 256:
            mc -= mc // 8
        return smem(nt, mc) <= optin

    lo, hi = 0, 65535
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if fits(mid) else (lo, mid - 1)
    return lo


@pytest.mark.parametrize("size", list(SIZES))
@pytest.mark.parametrize("checkers", ["fixed20", "shipped"])
def test_point_to_point_equals_oracle(gpu_ctx, size, checkers):
    tgt = _map(size)
    assert len(tgt) > _cta_limit(1500)
    prm, oprm = _params(**(FIXED20 if checkers == "fixed20" else {}))
    for n, seed in ((400, 1), (1500, 2)):
        src, T = _source(tgt, n, seed)
        gs = _guesses(T, 4, seed)
        res = _icp(prm).compute_batch(src, tgt, gs)
        for k, g in enumerate(gs):
            w = _assert_oracle(res, k, src, tgt, g, oprm)
        assert w["status"] == 0


def test_sizes_beyond_16_bit_indices():
    assert len(_map("80k")) > 65535 and len(_map("250k")) > 200000


def test_point_to_plane_equals_oracle(gpu_ctx):
    tgt = _map("30k")
    prm, oprm = _params(minimizer=1, normals_knn=5, **FIXED20)
    src, T = _source(tgt, 1000, 3)
    gs = _guesses(T, 3, 3)
    res = _icp(prm).compute_batch(src, tgt, gs)
    for k, g in enumerate(gs):
        _assert_oracle(res, k, src, tgt, g, oprm)


@pytest.mark.parametrize("delta", [0, 1])
def test_target_at_the_limit_and_one_past(gpu_ctx, delta):
    """At the limit one icp_kernel launch; one point past it the in-CTA launch (it takes the targets that fit, here
    none) plus the map class: build (nine launches) and icp_kernel's map class."""
    from sonar_slam_b200 import _lib
    ctx = _lib.default_context()
    src, T = _source(_map("80k"), 1500, 4)
    nt = _cta_limit(len(src)) + delta
    tgt = _map("80k")[:nt]
    assert len(tgt) == nt
    prm, oprm = _params(**FIXED20)
    gs = _guesses(T, 2, 4)
    n0 = ctx.launches
    res = _icp(prm).compute_batch(src, tgt, gs)
    assert ctx.launches - n0 == (1 if delta == 0 else 11)
    for k, g in enumerate(gs):
        _assert_oracle(res, k, src, tgt, g, oprm)


def test_mixed_batch(gpu_ctx):
    """Small and map targets in one compute_pairs call: all equal the oracle, and the small ones equal a call with
    only them."""
    rng = np.random.default_rng(9)
    pairs = []
    for c in range(6):
        s, t, T = synth.make_icp_pair(700 + c, n_source=800, n_target=3000)
        pairs.append((s, t, _guesses(T, 2, c)))
    big = _map("80k")
    for seed in (5, 6):
        s, T = _source(big, 1200, seed)
        pairs.insert(int(rng.integers(len(pairs))), (s, big, _guesses(T, 2, seed)))
    prm, oprm = _params()
    icp = _icp(prm)
    out = icp.compute_pairs([p[0] for p in pairs], [p[1] for p in pairs], [p[2] for p in pairs])
    small = [p for p in pairs if len(p[1]) < 10000]
    alone = icp.compute_pairs([p[0] for p in small], [p[1] for p in small], [p[2] for p in small])
    si = 0
    for (s, t, gs), r in zip(pairs, out):
        for k, g in enumerate(gs):
            _assert_oracle(r, k, s, t, g, oprm)
        if len(t) < 10000:
            for key in ("T", "iterations", "inliers", "status"):
                assert np.array_equal(r[key], alone[si][key])
            si += 1


def _oracle_icp_with_cov(src, tgt, guesses):
    """slam.py:346-371 restated with the oracle's ICP and scikit-learn's MinCovDet."""
    from sklearn.covariance import MinCovDet
    samples = []
    for g in guesses:
        r = orc.icp(src, tgt, g.matrix().astype(np.float32))
        if r["status"] == 0:
            T = r["T"]
            samples.append((T[0, 2], T[1, 2], np.arctan2(T[1, 0], T[0, 0])))
    samples = np.array(samples)
    fcov = MinCovDet(store_precision=False, support_fraction=0.8).fit(samples)
    return samples, fcov.location_


def test_slam_compute_icp_with_cov_on_a_map(gpu_ctx, icp_yaml):
    from sonar_slam_b200.bruce_slam.slam import SLAM, Pose2
    s = SLAM()
    s.icp.loadFromYaml(icp_yaml)
    tgt = _map("80k")
    problems = []
    for seed in (7, 8):
        src, T = _source(tgt, 1500, seed)
        th = np.arctan2(T[1, 0], T[0, 0])
        rng = np.random.default_rng(seed)
        problems.append((src, tgt, [Pose2(*(np.array([T[0, 2], T[1, 2], th]) + rng.normal(0, [0.2, 0.2, 0.02])))
                                    for _ in range(30)]))
    np.random.seed(21)
    want = [_oracle_icp_with_cov(*p) for p in problems]
    np.random.seed(21)
    one = [s.compute_icp_with_cov(*p) for p in problems]
    np.random.seed(21)
    batch = s.compute_icp_with_cov_batch(problems)
    for (ws, wloc), o, b in zip(want, one, batch):
        assert o[0] == "success" and b[0] == "success"
        assert np.array_equal(o[3], ws) and np.array_equal(b[3], ws)
        assert np.array_equal([o[1].x(), o[1].y(), o[1].theta()], wloc)
        assert np.allclose([b[1].x(), b[1].y(), b[1].theta()], wloc, rtol=1e-9, atol=1e-12)
        assert np.allclose(b[2], o[2], rtol=1e-9, atol=1e-12)


def _check_match(ref, pts, max_dist=10.0):
    from sonar_slam_b200.bruce_slam import pcl
    ids, d = pcl.match(ref, pts, 1, max_dist)
    wids, wd = orc.match(ref, pts, max_dist)
    assert np.array_equal(ids, wids) and np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    return ids


@pytest.mark.parametrize("size", ["30k", "250k"])
def test_match_equals_oracle(gpu_ctx, size):
    ref = _map(size)
    rng = np.random.default_rng(12)
    q = np.concatenate([ref[rng.integers(len(ref), size=3000)] + rng.normal(0, 0.3, (3000, 2)),
                        rng.uniform(ref.min(0) - 20, ref.max(0) + 20, (2000, 2))]).astype(np.float32)
    ids = _check_match(ref, q)
    assert (ids >= 0).sum() > 3000


def test_match_duplicates_lowest_index_wins(gpu_ctx):
    ref = _map("30k")
    dup = np.concatenate([ref, ref[::-1]]).astype(np.float32)  # every point twice, at i and 2n - 1 - i
    q = ref[::7] + np.float32(0.01)
    ids = _check_match(dup, q)
    assert (ids[0] < len(ref)).all()


@pytest.mark.parametrize("shape", ["line", "one_cell"])
def test_match_degenerate_reference(gpu_ctx, shape):
    rng = np.random.default_rng(13)
    n = 40000
    if shape == "line":
        t = rng.uniform(0, 500, n)
        ref = np.c_[t, 0.5 * t + 3.0]
    else:
        ref = 1.0 + rng.uniform(0, 0.01, (n, 2))
    ref = ref.astype(np.float32)
    q = (ref[rng.integers(n, size=2000)] + rng.normal(0, 0.5, (2000, 2))).astype(np.float32)
    _check_match(ref, q)


def _match_limit():
    """Largest reference match_kernel lays out: 8 B per point plus a cell table of 1.5 entries per point (at most
    16 384), next to the kernel's 672 B of static shared memory (icp.cu, match_cta_smem)."""
    import torch
    room = torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 672
    lo, hi = 0, 65535
    while lo < hi:
        mid = (lo + hi + 1) // 2
        mc = min(max(mid + mid // 2, 256), 16384)
        lo, hi = (mid, hi) if 8 * mid + 4 * ((mc + 2) // 2 + 1) + 16 <= room else (lo, mid - 1)
    return lo


@pytest.mark.parametrize("delta", [0, 1])
def test_match_at_the_limit_and_one_past(gpu_ctx, delta):
    """At the limit one match_kernel launch; one point past it that launch plus the map class (nine build launches
    and match_map_kernel)."""
    from sonar_slam_b200 import _lib
    ctx = _lib.default_context()
    ref = _map("80k")[: _match_limit() + delta]
    q = (ref[::5] + np.float32(0.05)).astype(np.float32)
    n0 = ctx.launches
    _check_match(ref, q)
    assert ctx.launches - n0 == (1 if delta == 0 else 11)


def test_device_flavour_shares_targets(gpu_ctx):
    """sfe_icp_dev (ops.icp) with a repeated tgt_id over two different map clouds and a small one: every problem equals
    the oracle, and equals the same batch with one private copy of its target per problem (null tgt_id)."""
    import torch
    from sonar_slam_b200 import ops
    small_s, small_t, small_T = synth.make_icp_pair(900, n_source=600, n_target=2500)
    tgts = [_map("80k"), _map("30k"), small_t]
    probs = []
    for k, ti in enumerate([1, 0, 2, 1, 0, 0, 2, 1]):
        if ti == 2:
            s, T = small_s, small_T
        else:
            s, T = _source(tgts[ti], 700 + 100 * k, 20 + k)
        probs.append((s, ti, _guesses(T, 1, 30 + k)[0]))
    prm, oprm = _params(**FIXED20)

    def pack(clouds):
        off = np.zeros(len(clouds) + 1, np.int32)
        off[1:] = np.cumsum([len(c) for c in clouds])
        return torch.from_numpy(np.concatenate(clouds)).cuda(), torch.from_numpy(off).cuda()

    spts, soff = pack([p[0] for p in probs])
    guess = torch.from_numpy(np.stack([p[2] for p in probs])).cuda()
    ns_max = max(len(p[0]) for p in probs)
    nt_max = max(len(t) for t in tgts)
    tpts, toff = pack(tgts)
    tid = torch.tensor([p[1] for p in probs], dtype=torch.int32).cuda()
    shared = ops.icp(spts, soff, tpts, toff, guess, ns_max, nt_max, params=prm, tgt_id=tid)
    cpts, coff = pack([tgts[p[1]] for p in probs])
    private = ops.icp(spts, soff, cpts, coff, guess, ns_max, nt_max, params=prm)
    torch.cuda.synchronize()
    a = {k: v.cpu().numpy() for k, v in shared.items()}
    b = {k: v.cpu().numpy() for k, v in private.items()}
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    for k, (s, ti, g) in enumerate(probs):
        _assert_oracle(a, k, s, tgts[ti], g, oprm)
