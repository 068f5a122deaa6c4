"""GPU: SurfaceNormalDataPointsFilter and ShadowDataPointsFilter on the reading cloud of an ICP call, bit for bit against
oracle/shadow_ref.c:

  * the normals stage alone (sfe_icp_surface_normals_dev): clouds of 0, 1, 2, knn - 1 and knn points, coincident
    points, lattices at the one-CTA limit and one past it, a 9 000-point cloud and a 243 k-point map;
  * ICP with the reading chain -- status, iterations, inliers and all nine entries of T: both minimisers, shipped and
    fixed-iteration checkers, eps values that remove nothing, most points or every point, octree and voxel filters
    before the normals, a robust filter, sampling normals on the reference, the in-CTA, map and global-source classes,
    the front end's size classes and FrontEnd.run_host, ops.icp with and without ids, ICP.compute, compute_batch and
    compute_pairs, and a context capped at one SM;
  * the C ABI's checks of the new kinds;
  * a sanity check, not a parity check: radial streaks are removed and walls seen head-on are kept.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import robust_ref
from oracle import shadow_ref as shr
from sonar_slam_b200 import _lib, ops, synth
from sonar_slam_b200.bruce_slam import pcl

pytestmark = pytest.mark.gpu
F32 = np.float32
MX, MN, OCT, VOX, SN = _lib.MAX_DIST, _lib.MIN_DIST, _lib.OCTREE, _lib.VOXEL, _lib.SAMPLING_NORMALS
NRM, SHD = _lib.NORMALS, _lib.SHADOW
CHECKERS = {"shipped": {}, "fixed20": dict(max_iterations=20, smooth_length=0)}
HALF_PI = float(F32(np.pi / 2))  # sinf = 1: no |n^ . p^| is above it, every point goes
SNRM_CTA_MAX = 4096


def _params(minimizer, knn=5, **kw):
    kw = dict(minimizer=minimizer, normals_knn=knn, **kw)
    return _lib.IcpParams(**kw), orc.IcpParams(**kw)


def _filters(**kw):
    return _lib.IcpFilters(**kw), shr.IcpFilters(**kw)


def _chain(eps=0.1, knn=5, before=(), after=()):
    return list(before) + [(NRM, knn, 0.0), (SHD, 0, eps)] + list(after)


def _same(got, want, what):
    assert (int(got["status"]), int(got["iterations"]), int(got["inliers"])) == \
        (want["status"], want["iterations"], want["inliers"]), what
    assert np.array_equal(np.asarray(got["T"], F32).view(np.uint32), np.asarray(want["T"], F32).view(np.uint32)), what


def _pack(clouds):
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    return torch.from_numpy(np.concatenate(clouds).astype(F32)).cuda(), torch.from_numpy(off).cuda()


def _run_dev(pairs, prm, flt, robust=None, ctx=None):
    srcs, tgts, gs = zip(*pairs)
    sp, so = _pack(srcs)
    tp, to = _pack(tgts)
    g = torch.from_numpy(np.stack(gs).astype(F32)).cuda()
    r = ops.icp(sp, so, tp, to, g, max(map(len, srcs)), max(map(len, tgts)), prm, filters=flt, robust=robust, ctx=ctx)
    torch.cuda.synchronize()
    return [dict(T=r["T"][k].cpu().numpy(), iterations=r["iterations"][k].item(), inliers=r["inliers"][k].item(),
                 status=r["status"][k].item()) for k in range(len(pairs))]


def _pairs(n=3, ns=400, nt=1400, seed=500):
    return [(s, t, T.astype(F32)) for k in range(n)
            for s, t, T in [synth.make_icp_pair(seed + k, n_source=ns, n_target=nt)]]


# ---------------------------------------------------------------- the normals stage alone
def _normals_dev(clouds, knn, ctx=None):
    clouds = [np.asarray(c, F32).reshape(-1, 2) for c in clouds]
    pts, off = _pack(clouds + [np.zeros((0, 2), F32)])
    off = off[:len(clouds) + 1].contiguous()
    out = ops.surface_normals(pts, off, max(1, max(len(c) for c in clouds)), knn, ctx=ctx)
    torch.cuda.synchronize()
    out, o = out.cpu().numpy(), off.cpu().numpy()
    return [out[o[c]:o[c + 1]] for c in range(len(clouds))]


def _normals_same(clouds, knn, ctx=None, what=""):
    got = _normals_dev(clouds, knn, ctx)
    for c, pts in enumerate(clouds):
        want = shr.reading_normals(pts, knn)
        assert np.array_equal(got[c].view(np.uint32), want.view(np.uint32)), (what, knn, c, len(pts))


def _lattice(n, spacing=0.1, seed=11):
    side = int(np.ceil(np.sqrt(n)))
    g = (np.stack(np.meshgrid(np.arange(side), np.arange(side)), -1).reshape(-1, 2) * spacing).astype(F32)
    return g[np.random.default_rng(seed).permutation(len(g))][:n]


@pytest.mark.parametrize("knn", [3, 5, 16])
def test_normals_stage_equals_oracle_around_the_one_cta_limit(knn):
    rng = np.random.default_rng(knn)
    small = [np.zeros((0, 2), F32), np.array([[1.0, 2.0]], F32), rng.normal(0, 2, (2, 2)).astype(F32),
             rng.normal(0, 2, (knn - 1, 2)).astype(F32), rng.normal(0, 2, (knn, 2)).astype(F32),
             np.tile(np.array([[0.5, -0.5]], F32), (40, 1)),
             np.repeat(rng.normal(0, 3, (30, 2)).astype(F32), 3, axis=0)]
    big = [_lattice(SNRM_CTA_MAX), _lattice(SNRM_CTA_MAX + 1, seed=12),
           synth.make_icp_pair(5, n_source=100, n_target=9000)[1]]
    _normals_same(small, knn, what="small")
    _normals_same(small + big, knn, what="with the map path")


def test_normals_stage_on_a_map_cloud():
    """(the oracle's brute-force neighbours take about two minutes on the map)"""
    big = synth.make_map_cloud(243_000, seed=3)[0]
    _normals_same([big, big[:2000]], 5, what="map")


def test_normals_stage_refusals():
    ctx = ops.context(0)
    pts, off = _pack([np.zeros((4, 2), F32)])
    for knn in (2, 17):
        with pytest.raises(_lib.SonarFEError, match="knn"):
            ops.surface_normals(pts, off, 4, knn, ctx=ctx)


# ---------------------------------------------------------------- the C ABI's checks
@pytest.mark.parametrize("bad", [
    dict(reference=[(NRM, 5, 0.0)]),
    dict(reference=[(SN, 1, np.inf), (SHD, 0, 0.1)]),
    dict(reading=[(SHD, 0, 0.1)]),
    dict(reading=[(SHD, 0, 0.1), (NRM, 5, 0.0)]),
    dict(reading=[(NRM, 2, 0.0)]),
    dict(reading=[(NRM, 17, 0.0)]),
    dict(reading=[(NRM, 5, 0.0), (NRM, 5, 0.0)]),
    dict(reading=[(NRM, 5, 0.0), (VOX, 1, 0.2)]),
    dict(reading=[(NRM, 5, 0.0), (OCT, 0, 0.2)]),
    dict(reading=[(NRM, 5, 0.0), (SHD, 0, np.inf)]),
    dict(reading=[(NRM, 5, 0.0), (SHD, 0, np.nan)]),
])
def test_set_filters_refusals_leave_the_setting(bad):
    ctx = ops.context(0)
    good = _lib.IcpFilters(reading=_chain())
    try:
        _lib.set_icp_filters(ctx, good)
        rc = ctx.lib.sfe_icp_set_filters(ctx.handle, ctypes.byref(_lib.IcpFilters(**bad)))
        assert rc != 0
        # the setting is the good chain still: a call runs it
        prm, oprm = _params(0)
        s, t, g = _pairs(1)[0]
        sp, so = _pack([s])
        tp, to = _pack([t])
        gd = torch.from_numpy(g[None]).cuda()
        T = torch.empty((1, 3, 3), dtype=torch.float32, device="cuda")
        it, inl, st = (torch.empty(1, dtype=torch.int32, device="cuda") for _ in range(3))
        p_ = lambda x: ctypes.c_void_p(x.data_ptr())  # noqa: E731
        _lib.check(ctx.lib.sfe_icp_dev(ctx.handle, ctypes.byref(prm), p_(sp), p_(so), p_(tp), p_(to), None, None, 1,
                                       len(s), len(t), p_(gd), p_(T), p_(it), p_(inl),
                                       p_(st)), "sfe_icp_dev")
        torch.cuda.synchronize()
        _same(dict(T=T[0].cpu().numpy(), iterations=it.item(), inliers=inl.item(), status=st.item()),
              shr.icp(s, t, g, oprm, shr.IcpFilters(reading=_chain())), bad)
    finally:
        _lib.set_icp_filters(ctx, None)


def test_frontend_refuses_a_bad_chain_and_3d_stays_unsupported():
    from oracle import featx_ref
    from sonar_slam_b200 import pipeline
    ctx = ops.context(0)
    d = synth.make_trajectory_frames(2, seed=3)
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    fe = pipeline.FrontEnd(ctx, maps, max_frames=4, min_points=30)
    rc = ctx.lib.sfe_frontend_set_icp_filters(fe.handle, ctypes.byref(_lib.IcpFilters(reading=[(SHD, 0, 0.1)])))
    assert rc != 0
    # 3-D clouds with any filter: SFE_ERR_UNSUPPORTED, nothing launched
    _lib.set_icp_filters(ctx, _lib.IcpFilters(reading=_chain()))
    try:
        prm = _lib.IcpParams()
        out = np.zeros(1, np.int32)
        assert ctx.lib.sfe_icp_source_limit(ctx.handle, ctypes.byref(prm), 3, _lib.ptr(out)) == -4  # SFE_ERR_UNSUPPORTED
    finally:
        _lib.set_icp_filters(ctx, None)


# ---------------------------------------------------------------- ICP with the reading chain
@pytest.mark.parametrize("checkers", list(CHECKERS))
@pytest.mark.parametrize("eps", [-0.1, 0.1, 1.4, HALF_PI])
@pytest.mark.parametrize("minimizer", [0, 1])
def test_icp_dev_equals_oracle(minimizer, eps, checkers):
    prm, oprm = _params(minimizer, **CHECKERS[checkers])
    flt, oflt = _filters(reading=_chain(eps))
    pairs = _pairs() + _pairs(1, 2000, 20000, seed=900)
    got = _run_dev(pairs, prm, flt)
    for k, (s, t, g) in enumerate(pairs):
        want = shr.icp(s, t, g, oprm, oflt)
        _same(got[k], want, (minimizer, eps, checkers, k))
        kept = len(shr.data_filters(s, _chain(eps)))
        if eps == HALF_PI:  # an emptied source: NO_OUTLIER with the trimmed filter on
            assert kept == 0 and want["status"] == 1
        elif eps < 0:
            assert kept == len(s)
        elif eps > 1:
            assert kept < len(s) / 2


def test_emptied_source_without_a_quantile_filter():
    prm, oprm = _params(0, trim_ratio=-1.0)
    flt, oflt = _filters(reading=_chain(HALF_PI))
    s, t, g = _pairs(1)[0]
    got = _run_dev([(s, t, g)], prm, flt)[0]
    want = shr.icp(s, t, g, oprm, oflt)
    _same(got, want, "emptied")
    assert want["status"] == 2  # NO_POINT


CHAINS = {
    "distance": dict(reading=_chain(0.2, 7, before=[(MX, -1, 28.0)], after=[(MN, -1, 1.0)])),
    "octree": dict(reading=_chain(0.15, 5, before=[(OCT, 2, 0.1)])),
    "voxel": dict(reading=_chain(0.3, 9, before=[(VOX, 1, 0.15)]), reference=[(VOX, 1, 0.1)]),
    "sampling_ref": dict(reading=_chain(0.1, 3), reference=[(MX, -1, 30.0), (SN, 1, np.inf)]),
    "outliers": dict(min_dist=0.01, median_factor=4.0, reading=_chain(0.2, 16)),
}


@pytest.mark.parametrize("robust", [None, "huber"])
@pytest.mark.parametrize("chain", list(CHAINS))
@pytest.mark.parametrize("minimizer", [0, 1])
def test_chains_and_robust(minimizer, chain, robust):
    prm, oprm = _params(minimizer, 7)
    flt, oflt = _filters(**CHAINS[chain])
    rb = _lib.IcpRobust(robust, 0.5) if robust else None
    orb = robust_ref.Robust(robust, 0.5) if robust else None
    pairs = _pairs(3, seed=600)
    got = _run_dev(pairs, prm, flt, rb)
    for k, (s, t, g) in enumerate(pairs):
        _same(got[k], shr.icp(s, t, g, oprm, oflt, orb), (minimizer, chain, robust, k))


@pytest.mark.parametrize("minimizer", [0, 1])
def test_map_and_global_source_classes(minimizer):
    """A 243 k-point map target (the map class) next to pipeline-sized problems, and a source above the shared-memory
    layouts (the global-source class; its normals on the map-grid path of the stage)"""
    big = synth.make_map_cloud(243_000, seed=3)[0]
    rng = np.random.default_rng(4)
    src = (big[rng.choice(len(big), 3000, replace=False)] - big.mean(0) + F32(0.05)).astype(F32)
    prm, oprm = _params(minimizer, 7)
    flt, oflt = _filters(reading=_chain(0.1))
    S = ops.icp_source_limit(2, prm, flt)
    assert S > SNRM_CTA_MAX
    g_big = np.array([[1, 0, big.mean(0)[0]], [0, 1, big.mean(0)[1]], [0, 0, 1]], F32)
    pairs = [(src, big.astype(F32), g_big)] + _pairs(1, S + 300, 20000, seed=950) + _pairs(2)
    got = _run_dev(pairs, prm, flt)
    for k, (s, t, g) in enumerate(pairs):
        _same(got[k], shr.icp(s, t, g, oprm, oflt), (minimizer, k))
    assert got[1]["status"] == 0


def test_ops_icp_with_ids_and_the_yaml_flavours():
    prm, oprm = _params(1, 7)
    flt, oflt = _filters(reading=_chain(0.2, 7, before=[(MX, -1, 28.0)]))
    base = _pairs(3, seed=1000)
    srcs, tgts = [p[0] for p in base], [p[1] for p in base[:2]]
    sid = np.array([0, 1, 2, 0, 2, 1], np.int32)
    tid = np.array([0, 1, 1, 0, 0, 1], np.int32)
    gs = np.stack([base[k % 3][2] for k in range(6)]).astype(F32)
    sp, so = _pack(srcs)
    tp, to = _pack(tgts)
    r = ops.icp(sp, so, tp, to, torch.from_numpy(gs).cuda(), max(map(len, srcs)), max(map(len, tgts)), prm,
                src_id=torch.from_numpy(sid).cuda(), tgt_id=torch.from_numpy(tid).cuda(), filters=flt)
    torch.cuda.synchronize()
    for k in range(6):
        got = dict(T=r["T"][k].cpu().numpy(), iterations=r["iterations"][k].item(), inliers=r["inliers"][k].item(),
                   status=r["status"][k].item())
        _same(got, shr.icp(srcs[sid[k]], tgts[tid[k]], gs[k], oprm, oflt), ("ids", k))

    text = ("readingDataPointsFilters:\n  - MaxDistDataPointsFilter: {maxDist: 28.0}\n"
            "  - SurfaceNormalDataPointsFilter: {knn: 7}\n  - ShadowDataPointsFilter: {eps: 0.2}\n"
            "referenceDataPointsFilters:\n  - SurfaceNormalDataPointsFilter: {knn: 7}\n"
            "matcher:\n  KDTreeMatcher:\n    maxDist: 10.0\noutlierFilters:\n  - TrimmedDistOutlierFilter: {ratio: 0.8}\n"
            "errorMinimizer:\n  PointToPlaneErrorMinimizer\n")
    icp = pcl.ICP()
    icp.params = pcl.parse_icp_yaml(text)
    oprm = orc.IcpParams(**{f: getattr(icp.params, f) for f, _ in _lib.IcpParams._fields_})
    for s, t, g in base:
        msg, T = icp.compute(s, t, g)
        want = shr.icp(s, t, g, oprm, oflt)
        assert msg == want["message"] and np.array_equal(T.view(np.uint32), np.asarray(want["T"], F32).view(np.uint32))
    s, t, _ = base[0]
    r = icp.compute_batch(s, t, gs)
    for k in range(len(gs)):
        want = shr.icp(s, t, gs[k], oprm, oflt)
        assert r["status"][k] == want["status"]
        assert np.array_equal(r["T"][k].view(np.uint32), np.asarray(want["T"], F32).view(np.uint32))
    r = icp.compute_pairs([p[0] for p in base], [p[1] for p in base], [[p[2], gs[3]] for p in base])
    for k, (s, t, g) in enumerate(base):
        for j, gg in enumerate((g, gs[3])):
            want = shr.icp(s, t, gg, oprm, oflt)
            assert np.array_equal(r[k]["T"][j].view(np.uint32), np.asarray(want["T"], F32).view(np.uint32)), (k, j)


def test_past_one_wave():
    """A context capped at one SM: the one-CTA normals stage and the data-filter pass take many clouds per CTA"""
    ctx = ops.context(0)
    ctx.set_grid_sms(1)
    try:
        clouds = [synth.make_icp_pair(40 + k, n_source=300 + 37 * k, n_target=10)[0] for k in range(40)]
        _normals_same(clouds, 5, ctx, "one SM")
        prm, oprm = _params(0)
        flt, oflt = _filters(reading=_chain(0.2))
        pairs = _pairs(24, 300, 900, seed=800)
        got = _run_dev(pairs, prm, flt, ctx=ctx)
        for k, (s, t, g) in enumerate(pairs):
            _same(got[k], shr.icp(s, t, g, oprm, oflt), ("one SM", k))
    finally:
        ctx.set_grid_sms(0)


@pytest.mark.parametrize("minimizer", [0, 1])
def test_frontend_size_classes_equal_oracle(minimizer):
    """sfe_frontend_icp_dev: frame-sized problems in the narrow / small class (the dense 64-register instantiations)
    and above it, the filters set on the context"""
    sizes = [(300, 420), (500, 700), (900, 1200), (1400, 2500)]
    prm, oprm = _params(minimizer, 7)
    flt, oflt = _filters(reading=_chain(0.15, 5, before=[(MX, -1, 30.0)]))
    probs = [(s, t, T.astype(F32)) for k, (ns, nt) in enumerate(sizes)
             for s, t, T in [synth.make_icp_pair(60 + k, n_source=ns, n_target=nt)]]
    P = len(probs)
    sp, so = _pack([p[0] for p in probs])
    tp, to = _pack([p[1] for p in probs])
    guess = torch.from_numpy(np.stack([p[2] for p in probs])).cuda()
    T = torch.empty((P, 3, 3), dtype=torch.float32, device="cuda")
    iters, inl, st = (torch.empty(P, dtype=torch.int32, device="cuda") for _ in range(3))
    ctx = ops.context(0)
    _lib.set_icp_filters(ctx, flt)
    p_ = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    try:
        _lib.check(ctx.lib.sfe_frontend_icp_dev(ctx.handle, ctypes.byref(prm), p_(sp), p_(so), p_(tp), p_(to), P,
                                                max(len(p[0]) for p in probs), max(len(p[1]) for p in probs),
                                                p_(guess), p_(T), p_(iters), p_(inl), p_(st), None),
                   "sfe_frontend_icp_dev")
        torch.cuda.synchronize()
    finally:
        _lib.set_icp_filters(ctx, None)
    ok = 0
    for k, (s, t, g) in enumerate(probs):
        got = dict(T=T[k].cpu().numpy(), iterations=iters[k].item(), inliers=inl[k].item(), status=st[k].item())
        want = shr.icp(s, t, g, oprm, oflt)
        _same(got, want, (minimizer, k))
        ok += want["status"] == 0
    assert ok >= 2


def test_frontend_run_equals_oracle_chain(monkeypatch):
    """FrontEnd(icp=IcpConfig(filters=...)) with the reading chain on every frame's cloud, frame for frame against
    oracle/pipeline_ref"""
    from oracle import featx_ref, pipeline_ref
    from sonar_slam_b200 import pipeline
    flt, oflt = _filters(reading=_chain(0.1, 5, before=[(MX, -1, 30.0)]))
    d = synth.make_trajectory_frames(10, seed=3)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    ctx = ops.context(0)
    maps = _lib.Maps(ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    fe = pipeline.FrontEnd(ctx, maps, max_frames=16, min_points=30, icp=_lib.IcpConfig(filters=flt))
    res = fe.run_host(frames, poses)
    monkeypatch.setattr(pipeline_ref.orc, "icp", lambda s, t, g, p: shr.icp(s, t, g, p, oflt))
    _, want = pipeline_ref.run(frames, poses, geo, min_points=30)
    ok = 0
    for i, w in enumerate(want):
        assert res["status"][i] == w["status"], i
        if w["status"] == 0:
            ok += 1
            _same(dict(T=res["T"][i], iterations=res["iterations"][i], inliers=res["inliers"][i], status=0), w, i)
    assert ok >= 5


# ---------------------------------------------------------------- sanity: what the filter is for
def test_radial_streaks_go_and_head_on_walls_stay():
    """Walls across the line of sight and radial streaks (one beam's detections smeared along the range axis): the
    device's normals with the shadow test keep the walls and drop the streaks; ICP with the chain equals the oracle"""
    rng = np.random.default_rng(9)
    walls, streaks = [], []
    for ang, rng_m in ((-0.5, 12.0), (0.0, 15.0), (0.45, 10.0)):  # wall segments facing the sensor
        u = np.linspace(-2.0, 2.0, 81)
        c, s = np.cos(ang), np.sin(ang)
        walls.append(np.stack([rng_m * c - u * s, rng_m * s + u * c], -1))
    for ang in (-0.25, 0.2, 0.7):  # radial streaks between the walls
        r = np.linspace(4.0, 8.0, 41)
        streaks.append(np.stack([r * np.cos(ang), r * np.sin(ang)], -1))
    walls = (np.concatenate(walls) + rng.normal(0, 0.005, (243, 2))).astype(F32)
    streaks = (np.concatenate(streaks) + rng.normal(0, 0.005, (123, 2))).astype(F32)
    cloud = np.concatenate([walls, streaks])
    n = _normals_dev([cloud], 5)[0]
    keep = np.array([shr.shadow_keep(x, y, nx, ny, 0.1) for (x, y), (nx, ny) in zip(cloud, n)])
    assert keep[:len(walls)].mean() > 0.95 and keep[len(walls):].mean() < 0.05
    kept = shr.data_filters(cloud, _chain(0.1))
    assert np.array_equal(kept, cloud[keep])
    prm, oprm = _params(0)
    flt, oflt = _filters(reading=_chain(0.1))
    g = np.array([[1, 0, 0.1], [0, 1, -0.05], [0, 0, 1]], F32)
    got = _run_dev([(cloud, walls, g)], prm, flt)[0]
    want = shr.icp(cloud, walls, g, oprm, oflt)
    _same(got, want, "streaks")
    assert want["status"] == 0 and want["inliers"] <= keep.sum()
