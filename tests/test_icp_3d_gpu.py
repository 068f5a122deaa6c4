"""3-D ICP on the device (`sfe_icp_dim_*`, `ops.icp` on [total,3], `pcl.ICP` on [N,3]) held to oracle/icp3_ref.c bit for
bit: status, iterations, inliers and all 16 entries of T."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import icp3_ref as o3, oracle as orc
from sonar_slam_b200 import _lib, ops, synth
from sonar_slam_b200.bruce_slam import pcl

pytestmark = pytest.mark.gpu
FIXED20 = dict(max_iterations=20, smooth_length=0)


def _packed(clouds, dim):
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    pts = np.concatenate([np.asarray(c, np.float32).reshape(-1, dim) for c in clouds] + [np.zeros((0, dim), np.float32)])
    return torch.from_numpy(np.ascontiguousarray(pts)).cuda(), torch.from_numpy(off).cuda(), max(map(len, clouds))


def _device(srcs, tgts, guesses, prm, src_id=None, tgt_id=None, dim=3):
    sp, so, ns = _packed(srcs, dim)
    tp, to, nt = _packed(tgts, dim)
    g = torch.from_numpy(np.ascontiguousarray(np.asarray(guesses, np.float32))).cuda()
    ids = lambda a: None if a is None else torch.from_numpy(np.asarray(a, np.int32)).cuda()
    out = ops.icp(sp, so, tp, to, g, ns, nt, _lib.IcpParams(**prm), src_id=ids(src_id), tgt_id=ids(tgt_id))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def _assert_exact(dev, want, what):
    bad = []
    for p, w in enumerate(want):
        same = (dev["status"][p] == w["status"] and dev["iterations"][p] == w["iterations"] and
                dev["inliers"][p] == w["inliers"] and dev["T"][p].tobytes() == np.float32(w["T"]).tobytes())
        if not same:
            bad.append((p, int(dev["status"][p]), w["status"], int(dev["iterations"][p]), w["iterations"],
                        int(dev["inliers"][p]), w["inliers"], float(np.abs(dev["T"][p] - w["T"]).max())))
    assert not bad, f"{what}: {len(bad)} of {len(want)} problems differ from the oracle, first {bad[:5]}"


def _oracle(srcs, tgts, guesses, prm, src_id=None, tgt_id=None):
    P = len(guesses)
    si = range(P) if src_id is None else src_id
    ti = range(P) if tgt_id is None else tgt_id
    return o3.icp3_many([(srcs[a], tgts[b], g) for a, b, g in zip(si, ti, guesses)], orc.IcpParams(**prm))


def _guess(rng, scale=1.0):
    T = synth.se3(rng.uniform(-0.3, 0.3, 3) * scale, rng.normal(size=3), rng.uniform(-0.05, 0.05) * scale)
    return T.astype(np.float32)


@pytest.fixture(scope="module")
def config3_pairs():
    rng = np.random.default_rng(11)
    pairs = [synth.make_icp_pair3(1000 + k) for k in range(200)]
    guesses = [np.eye(4, dtype=np.float32) if k % 2 == 0 else _guess(rng) for k in range(200)]
    return [p[0] for p in pairs], [p[1] for p in pairs], guesses


@pytest.mark.parametrize("prm", [FIXED20, {}], ids=["fixed20", "shipped_checkers"])
def test_config3_pairs_match_the_oracle(config3_pairs, prm):
    srcs, tgts, guesses = config3_pairs
    dev = _device(srcs, tgts, guesses, prm)
    _assert_exact(dev, _oracle(srcs, tgts, guesses, prm), f"config-3 pairs {prm}")
    assert (dev["status"] == 0).all()


def test_targets_at_the_cta_limit_and_one_above():
    ns = 1500
    limit = ops.icp_cta_limit(3, ns)
    assert 1000 < limit < 65535
    rng = np.random.default_rng(5)
    src, big, _ = synth.make_icp_pair3(7, n_source=ns, n_target=limit + 1)
    assert len(big) == limit + 1
    tgts = [big[:limit], big, big[:limit - 1]]
    guesses = [np.eye(4, dtype=np.float32), _guess(rng)]
    gl = [g for _ in tgts for g in guesses]
    tid = [t for t in range(len(tgts)) for _ in guesses]
    for prm in (FIXED20, {}):
        dev = _device([src], tgts, gl, prm, src_id=[0] * len(gl), tgt_id=tid)
        _assert_exact(dev, _oracle([src], tgts, gl, prm, [0] * len(gl), tid), f"limit {limit} {prm}")


@pytest.mark.parametrize("n_target", [100_000, 250_000])
def test_map_class_targets_with_30_guesses(n_target):
    rng = np.random.default_rng(n_target)
    src, tgt, _ = synth.make_icp_pair3(3, n_source=1500, n_target=n_target, extent=150.0)
    guesses = np.stack([np.eye(4, dtype=np.float32)] + [_guess(rng) for _ in range(29)])
    icp = pcl.ICP()
    icp.params = _lib.IcpParams()
    res = icp.compute_batch(src, tgt, guesses)
    want = o3.icp3_many([(src, tgt, g) for g in guesses])
    _assert_exact(res, want, f"{n_target}-point target")
    msg, T = icp.compute(src, tgt, guesses[3])
    assert msg == want[3]["message"] and T.tobytes() == want[3]["T"].tobytes()


def test_packed_batch_mixes_both_classes():
    rng = np.random.default_rng(8)
    pairs = [synth.make_icp_pair3(50 + k, n_source=800 + 300 * k, n_target=n)
             for k, n in enumerate([3000, 120_000, 12_000, 60_000])]
    srcs, tgts = [p[0] for p in pairs], [p[1] for p in pairs]
    gs = [[np.eye(4, dtype=np.float32), _guess(rng)] for _ in pairs]
    icp = pcl.ICP()
    icp.params = _lib.IcpParams()
    res = icp.compute_pairs(srcs, tgts, gs)
    for k, r in enumerate(res):
        _assert_exact(r, o3.icp3_many([(srcs[k], tgts[k], g) for g in gs[k]]), f"compute_pairs pair {k}")
    flat = [g for gg in gs for g in gg]
    sid = [k for k in range(len(pairs)) for _ in range(2)]
    dev = _device(srcs, tgts, flat, FIXED20, src_id=sid, tgt_id=sid)
    _assert_exact(dev, _oracle(srcs, tgts, flat, FIXED20, sid, sid), "ops.icp mixed classes")


def test_columns_ties_and_points_at_max_dist():
    rng = np.random.default_rng(9)
    # a tall column: 0.4 m x 0.4 m footprint, 30 m of z
    col = np.c_[rng.uniform(0, 0.4, (6000, 2)), rng.uniform(0, 30, 6000)].astype(np.float32)
    col_src = (col[rng.choice(6000, 1200, replace=False)] @ synth.se3([0.05, -0.02, 0.3], [0, 0, 1], 0.02)[:3, :3].T
               + np.float32([0.02, 0.01, 0.4])).astype(np.float32)
    # coincident points and ties: a 0.25 m lattice, every point twice; sources on a 0.125 m lattice
    lat = (np.round(rng.uniform(-3, 3, (2500, 3)) * 4) / 4).astype(np.float32)
    dup = np.r_[lat, lat].astype(np.float32)
    dup_src = (np.round(rng.uniform(-3, 3, (900, 3)) * 8) / 8).astype(np.float32)
    # points at exactly maxDist (2 m: integer lattice, sources 2 m above it), and some farther
    grid = np.stack(np.meshgrid(np.arange(0, 20.0, 4), np.arange(0, 20.0, 4), [0.0]), -1).reshape(-1, 3).astype(np.float32)
    at_max = np.r_[grid + np.float32([0, 0, 2]), grid[:10] + np.float32([0, 0, 2.5])].astype(np.float32)
    srcs, tgts = [col_src, dup_src, at_max], [col, dup, grid]
    I = np.eye(4, dtype=np.float32)
    for prm in (FIXED20, {}, dict(matcher_max_dist=2.0, outlier_max_dist=-1.0, trim_ratio=-1.0, max_iterations=1),
                dict(matcher_max_dist=2.0, outlier_max_dist=2.0, flags=1, max_iterations=3)):
        dev = _device(srcs, tgts, [I, I, I], prm)
        _assert_exact(dev, _oracle(srcs, tgts, [I, I, I], prm), f"special clouds {prm}")
    dev = _device(srcs, tgts, [I] * 3, dict(matcher_max_dist=2.0, trim_ratio=-1.0, outlier_max_dist=-1.0,
                                            max_iterations=1))
    assert dev["inliers"][2] == len(grid)  # the points at exactly 2 m count, the ones at 2.5 m do not


def test_planar_clouds_and_the_2d_path():
    pairs = [synth.make_icp_pair(300 + k) for k in range(16)]
    s2, t2 = [p[0] for p in pairs], [p[1] for p in pairs]
    z = lambda c: np.c_[c, np.zeros(len(c), np.float32)].astype(np.float32)
    I3, I4 = np.eye(3, dtype=np.float32), np.eye(4, dtype=np.float32)
    dev3 = _device([z(c) for c in s2], [z(c) for c in t2], [I4] * 16, {})
    _assert_exact(dev3, _oracle([z(c) for c in s2], [z(c) for c in t2], [I4] * 16, {}), "z = 0 clouds")
    dev2 = _device(s2, t2, [I3] * 16, {}, dim=2)
    want2 = [orc.icp(a, b) for a, b in zip(s2, t2)]
    for p, w in enumerate(want2):  # the 2-D device path equals its oracle, so the two relate as the oracles do
        assert dev2["status"][p] == w["status"] and dev2["T"][p].tobytes() == w["T"].tobytes()
        assert (dev3["T"][p][2] == [0, 0, 1, 0]).all()
    # dim 2 through sfe_icp_dim_dev: sfe_icp_dev's launches and results
    sp, so, ns = _packed(s2, 2)
    tp, to, nt = _packed(t2, 2)
    g = torch.from_numpy(np.stack([I3] * 16)).cuda()
    ctx = ops.context(0)
    prm = _lib.IcpParams()
    outs = []
    for fn, extra in (("sfe_icp_dev", ()), ("sfe_icp_dim_dev", (2,))):
        T = torch.empty((16, 3, 3), device="cuda")
        r = [torch.empty(16, dtype=torch.int32, device="cuda") for _ in range(3)]
        n0 = ctx.lib.sfe_launch_count(ctx.handle)
        args = (ctx.handle, ctypes.byref(prm), ops._dp(sp), ops._dp(so), ops._dp(tp), ops._dp(to), None, None, 16)
        _lib.check(getattr(ctx.lib, fn)(*args, *extra, ns, nt, ops._dp(g), ops._dp(T), *map(ops._dp, r)), fn)
        torch.cuda.synchronize()
        outs.append((ctx.lib.sfe_launch_count(ctx.handle) - n0, T.cpu().numpy().tobytes(), [x.cpu().numpy().tolist() for x in r]))
    assert outs[0] == outs[1]


def test_statuses_and_rejections_on_the_device():
    src, tgt, _ = synth.make_icp_pair3(21, n_source=500, n_target=4000)
    bad = np.eye(4, dtype=np.float32)
    bad[1, 1] = 1.5
    I = np.eye(4, dtype=np.float32)
    srcs, tgts = [src, src, src + np.float32(200)], [np.zeros((0, 3), np.float32), tgt, tgt]
    prm = {}
    dev = _device(srcs, tgts, [I, bad, I], prm)
    _assert_exact(dev, _oracle(srcs, tgts, [I, bad, I], prm), "statuses")
    assert dev["status"].tolist() == [6, 5, 1]
    icp = pcl.ICP()
    icp.params = _lib.IcpParams()
    with pytest.raises(RuntimeError, match="not orthogonal"):
        icp.compute(src, tgt, bad)
    with pytest.raises(RuntimeError, match="empty"):
        icp.compute(src, np.zeros((0, 3), np.float32), I)
    # what the 3-D chain does not run is refused on the device side too, before any launch
    ctx = ops.context(0)
    sp, so, ns = _packed([src], 3)
    tp, to, nt = _packed([tgt], 3)
    g = torch.from_numpy(I[None]).cuda()
    T = torch.empty((1, 4, 4), device="cuda")
    r = [torch.empty(1, dtype=torch.int32, device="cuda") for _ in range(3)]
    for p in (_lib.IcpParams(minimizer=1), _lib.IcpParams(flags=2)):
        n0 = ctx.lib.sfe_launch_count(ctx.handle)
        rc = ctx.lib.sfe_icp_dim_dev(ctx.handle, ctypes.byref(p), ops._dp(sp), ops._dp(so), ops._dp(tp), ops._dp(to),
                                     None, None, 1, 3, ns, nt, ops._dp(g), ops._dp(T), *map(ops._dp, r))
        assert rc != 0 and b"not supported" in ctx.lib.sfe_last_error()
        assert ctx.lib.sfe_launch_count(ctx.handle) == n0
    _lib.set_icp_filters(ctx, _lib.IcpFilters(min_dist=0.1))
    try:
        rc = ctx.lib.sfe_icp_dim_dev(ctx.handle, ctypes.byref(_lib.IcpParams()), ops._dp(sp), ops._dp(so), ops._dp(tp),
                                     ops._dp(to), None, None, 1, 3, ns, nt, ops._dp(g), ops._dp(T), *map(ops._dp, r))
        assert rc != 0 and b"filters" in ctx.lib.sfe_last_error()
        assert ctx.lib.sfe_icp_dim_dev(ctx.handle, ctypes.byref(_lib.IcpParams()), ops._dp(sp), ops._dp(so),
                                       ops._dp(tp), ops._dp(to), None, None, 1, 4, ns, nt, ops._dp(g), ops._dp(T),
                                       *map(ops._dp, r)) != 0
    finally:
        _lib.set_icp_filters(ctx, None)
