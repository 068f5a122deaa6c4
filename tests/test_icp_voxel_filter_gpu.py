"""GPU: VoxelGridDataPointsFilter in the ICP data-filter chains, bit for bit against oracle/voxel_filter_ref.c --
status, iterations, inliers and all nine entries of T:

  * the filter on either cloud, alone and mixed with the octree and distance filters, point-to-point and
    point-to-plane (a reference voxel filter before the normals), on pipeline-sized and config-3 pairs;
  * compute (one guess), compute_batch (ids: the clouds filtered once per problem) and compute_pairs (once per cloud),
    in one call whose targets take the in-CTA and the map class and whose sources take the shared-memory and the
    global-source class, at the class bounds measured on the filtered clouds;
  * the front end's size classes (sfe_frontend_icp_dev) and the batched front end against the oracle chain;
  * all points in one voxel, a filter chain that empties a cloud, clouds given empty to compute, a long voxel at
    x = -0.0, more than 65 535 clouds filtered in one call, and the voxel-count overflow, refused before the ICP
    launch.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import voxel_filter_ref as vfr
from sonar_slam_b200 import _lib, ops, synth
from sonar_slam_b200.bruce_slam import pcl

pytestmark = pytest.mark.gpu
F32 = np.float32
MX, MN, OCT, VOX = _lib.MAX_DIST, _lib.MIN_DIST, _lib.OCTREE, _lib.VOXEL

CHAINS = {
    "reading": dict(reading=[(VOX, 1, 0.3)]),
    "reading_mixed": dict(reading=[(MX, -1, 18.0), (VOX, 1, 0.25), (OCT, 2, 0.5)]),
    "reference": dict(reference=[(VOX, 1, 0.2)]),
    "reference_mixed": dict(reference=[(OCT, 0, 0.1), (VOX, 1, 0.3), (MN, 0, -8.0), (VOX, 1, 0.45)]),
    "both": dict(min_dist=0.01, reading=[(VOX, 1, 0.2), (MX, 1, 15.0)], reference=[(MX, -1, 25.0), (VOX, 1, 0.15)]),
}
CHECKERS = {"shipped": {}, "fixed20": dict(max_iterations=20, smooth_length=0)}


def _filters(kw):
    return _lib.IcpFilters(**kw), vfr.IcpFilters(**kw)


def _params(minimizer=0, **kw):
    kw = dict(minimizer=minimizer, normals_knn=5, **kw)
    return _lib.IcpParams(**kw), orc.IcpParams(**kw)


def _same(got, want, what):
    assert (int(got["status"]), int(got["iterations"]), int(got["inliers"])) == \
        (want["status"], want["iterations"], want["inliers"]), what
    assert np.array_equal(np.asarray(got["T"], F32).view(np.uint32), np.asarray(want["T"], F32).view(np.uint32)), what


def _pack(clouds):
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    return torch.from_numpy(np.concatenate(clouds).astype(F32)).cuda(), torch.from_numpy(off).cuda()


def _rows(r, P):
    return [dict(T=r["T"][k].cpu().numpy(), iterations=r["iterations"][k].item(), inliers=r["inliers"][k].item(),
                 status=r["status"][k].item()) for k in range(P)]


def _run_dev(pairs, prm, flt, ctx=None):
    srcs, tgts, gs = zip(*pairs)
    sp, so = _pack(srcs)
    tp, to = _pack(tgts)
    g = torch.from_numpy(np.stack(gs).astype(F32)).cuda()
    r = ops.icp(sp, so, tp, to, g, max(map(len, srcs)), max(map(len, tgts)), prm, filters=flt, ctx=ctx)
    torch.cuda.synchronize()
    return _rows(r, len(pairs))


def _pairs(kind, n=3):
    size = dict(pipeline=(400, 1400), config3=(2000, 20000))[kind]
    out = []
    for seed in range(n):
        s, t, T = synth.make_icp_pair(500 + seed, n_source=size[0], n_target=size[1])
        out.append((s, t, T.astype(F32)))
    return out


@pytest.mark.parametrize("checkers", list(CHECKERS))
@pytest.mark.parametrize("chain", list(CHAINS))
@pytest.mark.parametrize("minimizer", [0, 1])
@pytest.mark.parametrize("kind", ["pipeline", "config3"])
def test_icp_dev_equals_oracle(kind, minimizer, chain, checkers):
    flt, oflt = _filters(CHAINS[chain])
    prm, oprm = _params(minimizer, **CHECKERS[checkers])
    pairs = _pairs(kind)
    got = _run_dev(pairs, prm, flt)
    for k, (s, t, g) in enumerate(pairs):
        want = vfr.icp(s, t, g, oprm, oflt)
        _same(got[k], want, (kind, minimizer, chain, checkers, k))


def test_plane_yaml_with_a_reference_voxel_filter_before_the_normals():
    text = ("readingDataPointsFilters:\n  - VoxelGridDataPointsFilter: {vSizeX: 0.2, vSizeY: 0.2}\n"
            "referenceDataPointsFilters:\n  - VoxelGridDataPointsFilter: {vSizeX: 0.15, vSizeY: 0.15}\n"
            "  - SurfaceNormalDataPointsFilter: {knn: 5}\n"
            "matcher:\n  KDTreeMatcher:\n    maxDist: 10.0\nerrorMinimizer:\n  PointToPlaneErrorMinimizer\n")
    icp = pcl.ICP()
    icp.params = pcl.parse_icp_yaml(text)
    assert icp.params.minimizer == 1
    oflt = vfr.IcpFilters(reading=[(VOX, 1, np.float32(0.2))], reference=[(VOX, 1, np.float32(0.15))])
    oprm = orc.IcpParams(**{f: getattr(icp.params, f) for f, _ in _lib.IcpParams._fields_})
    ok = 0
    for s, t, g in _pairs("config3", 2):
        msg, T = icp.compute(s, t, g)
        want = vfr.icp(s, t, g, oprm, oflt)
        assert msg == want["message"]
        assert np.array_equal(T.view(np.uint32), np.asarray(want["T"], F32).view(np.uint32))
        ok += want["status"] == 0
    assert ok >= 1


def _bounds(minimizer, vs):
    """Clouds whose filtered sizes sit on the class bounds: S (the source limit) and L (the in-CTA target limit next to
    S-point sources).  A lattice with one point per voxel keeps every point, in its order."""
    prm, _ = _params(minimizer, trim_ratio=0.8)
    flt = _lib.IcpFilters(reading=[(VOX, 1, vs)], reference=[(VOX, 1, vs)])
    S = ops.icp_source_limit(2, prm, flt)
    L = ops.icp_cta_limit(2, S)
    return S, L


def _lattice_cloud(n, seed, pitch):
    """n points of a noisy wall scene snapped to the voxel centres of a `pitch` grid, one point per voxel."""
    s, _, _ = synth.make_icp_pair(seed, n_source=4 * n, n_target=100, extent=max(40.0, pitch * np.sqrt(n) * 2))
    q = np.unique(np.floor(s / pitch).astype(np.int64), axis=0)
    rng = np.random.default_rng(seed)
    q = q[rng.permutation(len(q))]
    if len(q) < n:  # top up with a far block of free voxels
        extra = np.stack(np.meshgrid(np.arange(400), np.arange(400)), -1).reshape(-1, 2) + q.max(0) + 10
        q = np.concatenate([q, extra[:n - len(q)]])
    return ((q[:n] + 0.5) * pitch).astype(F32)


@pytest.mark.parametrize("minimizer", [0, 1])
def test_compute_batch_and_pairs_across_launch_classes(minimizer):
    """compute (one guess), compute_batch (ids: filtered once per problem) and compute_pairs (once per cloud) with the
    filtered sources at S and S + 1 and the filtered targets at L and L + 1, plus a raw map-sized target the filter
    thins into the in-CTA class."""
    vs = 0.25
    S, L = _bounds(minimizer, vs)
    prm, oprm = _params(minimizer, trim_ratio=0.8)
    kw = dict(reading=[(VOX, 1, vs)], reference=[(VOX, 1, vs)])
    flt, oflt = _filters(kw)
    icp = pcl.ICP()
    icp.params = _lib.IcpConfig(trim_ratio=0.8, minimizer=minimizer, normals_knn=5, filters=flt)
    srcs = [_lattice_cloud(S, 1, vs), _lattice_cloud(S + 1, 2, vs)]
    tgts = [_lattice_cloud(L, 3, vs), _lattice_cloud(L + 1, 4, vs)]
    for c in srcs + tgts:  # the filter keeps every point of these clouds, so the sizes are the filtered ones
        assert np.array_equal(vfr.voxel_filter(c, vs), c)
    shift = np.array([[1, 0, 0.1], [0, 1, -0.05], [0, 0, 1]], F32)
    gs = [np.eye(3, dtype=F32), shift]
    # compute and compute_batch on one pair of every class
    for s in srcs:
        for t in tgts:
            msg, T = icp.compute(s, t, gs[1])
            want = vfr.icp(s, t, gs[1], oprm, oflt)
            assert msg == want["message"] and np.array_equal(T.view(np.uint32), want["T"].view(np.uint32))
    res = icp.compute_batch(srcs[1], tgts[1], gs)
    for j, g in enumerate(gs):
        got = dict(T=res["T"][j], iterations=res["iterations"][j], inliers=res["inliers"][j], status=res["status"][j])
        _same(got, vfr.icp(srcs[1], tgts[1], g, oprm, oflt), ("batch", j))
    # compute_pairs: every source against every target, and a map-sized raw target
    _, big, _ = synth.make_icp_pair(9, n_source=100, n_target=60000, extent=120.0)
    assert len(big) > L + 1
    pairs = [(s, t) for s in srcs for t in tgts + [big]]
    res = icp.compute_pairs([p[0] for p in pairs], [p[1] for p in pairs], [gs] * len(pairs))
    for k, (s, t) in enumerate(pairs):
        for j, g in enumerate(gs):
            got = dict(T=res[k]["T"][j], iterations=res[k]["iterations"][j], inliers=res[k]["inliers"][j],
                       status=res[k]["status"][j])
            _same(got, vfr.icp(s, t, g, oprm, oflt), ("pairs", k, j))


@pytest.mark.parametrize("ids", [False, True])
def test_ops_icp_with_and_without_ids_equals_oracle(ids):
    flt, oflt = _filters(CHAINS["both"])
    prm, oprm = _params(0)
    pairs = _pairs("pipeline", 2)
    srcs, tgts = [p[0] for p in pairs], [p[1] for p in pairs]
    shift = np.array([[1, 0, 0.1], [0, 1, 0.05], [0, 0, 1]], F32)
    sid, tid = ([0, 1, 0, 1], [0, 1, 1, 0]) if ids else ([0, 1], [0, 1])
    gs = [(pairs[t][2] @ (shift if k >= 2 else np.eye(3, dtype=F32))).astype(F32) for k, t in enumerate(tid)]
    if ids:
        sp, so = _pack(srcs)
        tp, to = _pack(tgts)
        r = ops.icp(sp, so, tp, to, torch.from_numpy(np.stack(gs)).cuda(), max(map(len, srcs)), max(map(len, tgts)),
                    prm, src_id=torch.tensor(sid, dtype=torch.int32, device="cuda"),
                    tgt_id=torch.tensor(tid, dtype=torch.int32, device="cuda"), filters=flt)
        torch.cuda.synchronize()
        got = _rows(r, len(gs))
    else:
        got = _run_dev([(srcs[k], tgts[k], gs[k]) for k in range(2)], prm, flt)
    for k in range(len(gs)):
        _same(got[k], vfr.icp(srcs[sid[k]], tgts[tid[k]], gs[k], oprm, oflt), (ids, k))


@pytest.mark.parametrize("setting", ["point", "plane"])
def test_frontend_size_classes_equal_oracle(setting):
    """sfe_frontend_icp_dev: frame-sized problems in the narrow / small class and above it, the voxel filter on both
    clouds (ICP filters set on the context)."""
    sizes = [(300, 420), (500, 700), (900, 1200), (1400, 2500)]
    kw = dict(reading=[(VOX, 1, 0.2)], reference=[(MX, -1, 30.0), (VOX, 1, 0.15)])
    flt, oflt = _filters(kw)
    prm, oprm = _params(1 if setting == "plane" else 0)
    probs = []
    for k, (ns, nt) in enumerate(sizes):
        s, t, T = synth.make_icp_pair(60 + k, n_source=ns, n_target=nt)
        probs.append((s, t, T.astype(F32)))
    P = len(probs)
    dev = "cuda:0"
    src = torch.from_numpy(np.concatenate([p[0] for p in probs])).to(dev)
    tgt = torch.from_numpy(np.concatenate([p[1] for p in probs])).to(dev)
    soff = torch.tensor(np.cumsum([0] + [len(p[0]) for p in probs]), dtype=torch.int32, device=dev)
    toff = torch.tensor(np.cumsum([0] + [len(p[1]) for p in probs]), dtype=torch.int32, device=dev)
    guess = torch.from_numpy(np.stack([p[2] for p in probs])).to(dev)
    T = torch.empty((P, 3, 3), dtype=torch.float32, device=dev)
    iters, inl, st = (torch.empty(P, dtype=torch.int32, device=dev) for _ in range(3))
    ctx = ops.context(0)
    _lib.set_icp_filters(ctx, flt)
    p_ = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    try:
        _lib.check(ctx.lib.sfe_frontend_icp_dev(ctx.handle, ctypes.byref(prm), p_(src), p_(soff), p_(tgt), p_(toff), P,
                                                max(len(p[0]) for p in probs), max(len(p[1]) for p in probs),
                                                p_(guess), p_(T), p_(iters), p_(inl), p_(st), None),
                   "sfe_frontend_icp_dev")
        torch.cuda.synchronize()
    finally:
        _lib.set_icp_filters(ctx, None)
    ok = 0
    for k, (s, t, g) in enumerate(probs):
        got = dict(T=T[k].cpu().numpy(), iterations=iters[k].item(), inliers=inl[k].item(), status=st[k].item())
        want = vfr.icp(s, t, g, oprm, oflt)
        _same(got, want, (setting, k))
        ok += want["status"] == 0
    assert ok >= 2


def test_frontend_run_equals_oracle_chain(monkeypatch):
    """FrontEnd(icp=IcpConfig(filters=...)) with voxel filters: frame clouds as readings, window submaps as
    references, frame for frame against oracle/pipeline_ref."""
    from oracle import featx_ref, pipeline_ref
    from sonar_slam_b200 import pipeline
    flt, oflt = _filters(dict(reading=[(VOX, 1, 0.4)], reference=[(MX, -1, 30.0), (VOX, 1, 0.3)]))
    d = synth.make_trajectory_frames(10, seed=3)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    ctx = ops.context(0)
    maps = _lib.Maps(ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    fe = pipeline.FrontEnd(ctx, maps, max_frames=16, min_points=30, icp=_lib.IcpConfig(filters=flt))
    res = fe.run_host(frames, poses)
    monkeypatch.setattr(pipeline_ref.orc, "icp", lambda s, t, g, p: vfr.icp(s, t, g, p, oflt))
    _, want = pipeline_ref.run(frames, poses, geo, min_points=30)
    ok = 0
    for i, w in enumerate(want):
        assert res["status"][i] == w["status"], i
        if w["status"] == 0:
            ok += 1
            got = dict(T=res["T"][i], iterations=res["iterations"][i], inliers=res["inliers"][i], status=0)
            _same(got, w, i)
    assert ok >= 5


@pytest.mark.parametrize("case", ["one_voxel_source", "one_voxel_target", "empty_source", "empty_target",
                                  "map_in_one_voxel"])
def test_clouds_in_one_voxel_or_emptied(case):
    """A voxel larger than the cloud leaves one point, its centroid; a distance filter before it can leave none (an
    emptied target is SFE_ICP_EMPTY_REF, an emptied source "no outlier to filter").  A map-sized target in one voxel
    takes the long-segment path (one warp's sequential sums)."""
    kw = dict(one_voxel_source=dict(reading=[(VOX, 1, 1e4)]),
              one_voxel_target=dict(reference=[(VOX, 1, 1e4)]),
              empty_source=dict(reading=[(MX, -1, 0.0), (VOX, 1, 0.2)]),
              empty_target=dict(reference=[(MX, -1, 0.0), (VOX, 1, 0.2)]),
              map_in_one_voxel=dict(reference=[(VOX, 1, 1e4)]))[case]
    flt, oflt = _filters(kw)
    prm, oprm = _params(0)
    if case == "map_in_one_voxel":
        s, t, T = synth.make_icp_pair(77, n_source=800, n_target=250000, extent=150.0)
        pairs = [(s, t, T.astype(F32))]
    else:
        pairs = _pairs("pipeline", 2)
    got = _run_dev(pairs, prm, flt)
    for k, (s, t, g) in enumerate(pairs):
        want = vfr.icp(s, t, g, oprm, oflt)
        _same(got[k], want, (case, k))
        if case == "empty_target":
            assert want["status"] == 6
        if case == "empty_source":
            assert want["status"] == 1


@pytest.mark.parametrize("side", ["reading", "reference"])
def test_voxel_count_overflow_is_refused_before_the_icp_launch(side):
    """A 0.01 m voxel over a 1 km cloud would need 10^10 voxels: upstream's 32-bit index would wrap.  The call fails
    with the message after the filter stages' launches and before any ICP launch: the results are left untouched."""
    s, t, T = _pairs("pipeline", 1)[0]
    far = np.array([[1000.0, 1000.0]], F32)
    s, t = (np.concatenate([s, far]), t) if side == "reading" else (s, np.concatenate([t, far]))
    kw = {side: [(VOX, 1, 0.01)]}
    flt, oflt = _filters(kw)
    with pytest.raises(vfr.VoxelOverflow):
        vfr.icp(s, t, T, orc.IcpParams(), oflt)
    ctx = ops.context(0)
    sp, so = _pack([s])
    tp, to = _pack([t])
    g = torch.from_numpy(T[None]).cuda()
    prm = _lib.IcpParams()
    before = ctx.launches
    with pytest.raises(_lib.SonarFEError, match="VoxelGridDataPointsFilter"):
        ops.icp(sp, so, tp, to, g, len(s), len(t), prm, filters=flt, ctx=ctx)
    stage_launches = ctx.launches - before
    assert 0 < stage_launches <= 9  # the compaction pass, the voxel stage's seven, the size restore: no ICP launch
    # the same call without the far point runs, and makes the stage launches plus the ICP's
    s2, t2 = (s[:-1], t) if side == "reading" else (s, t[:-1])
    sp2, so2 = _pack([s2])
    tp2, to2 = _pack([t2])
    before = ctx.launches
    r2 = ops.icp(sp2, so2, tp2, to2, g, len(s2), len(t2), prm, filters=flt, ctx=ctx)
    torch.cuda.synchronize()
    assert ctx.launches - before > stage_launches
    _same(_rows(r2, 1)[0], vfr.icp(s2, t2, T, orc.IcpParams(), oflt), side)


@pytest.mark.parametrize("case", ["empty_source", "empty_target"])
def test_compute_with_an_empty_cloud(case):
    """pcl.ICP.compute on a cloud given empty (ns_max or nt_max 0) with voxel filters on both clouds: the oracle's
    message ("no outlier to filter" for the source), or its exception for an empty reference, as without a filter."""
    flt, oflt = _filters(dict(reading=[(VOX, 1, 0.2)], reference=[(VOX, 1, 0.2)]))
    s, t, g = _pairs("pipeline", 1)[0]
    if case == "empty_source":
        s = np.zeros((0, 2), F32)
    else:
        t = np.zeros((0, 2), F32)
    icp = pcl.ICP()
    icp.params = _lib.IcpConfig(filters=flt)
    want = vfr.icp(s, t, g, orc.IcpParams(), oflt)
    if want["status"] in (5, 6):
        with pytest.raises(RuntimeError, match=want["message"]):
            icp.compute(s, t, g)
    else:
        msg, T = icp.compute(s, t, g)
        assert msg == want["message"] and np.array_equal(T.view(np.uint32), want["T"].view(np.uint32))
    assert want["status"] == (6 if case == "empty_target" else 1)


@pytest.mark.parametrize("side", ["reading", "reference"])
def test_long_voxel_at_negative_zero(side):
    """A voxel of 300 points (the warp-summed path) whose x are all -0.0, in a cloud with other voxels."""
    s, t, g = _pairs("pipeline", 1)[0]
    rng = np.random.default_rng(4)
    wall = np.c_[np.full(300, -0.0), rng.uniform(60.0, 60.15, 300)].astype(F32)  # a voxel of its own
    cloud = np.concatenate([s if side == "reading" else t, wall]).astype(F32)
    kept = vfr.voxel_filter(cloud, 0.2)
    assert (kept[:, 0].view(np.uint32) == 0x80000000).sum() >= 1
    s, t = (cloud, t) if side == "reading" else (s, cloud)
    flt, oflt = _filters({side: [(VOX, 1, 0.2)]})
    prm, oprm = _params(0)
    got = _run_dev([(s, t, g)], prm, flt)
    _same(got[0], vfr.icp(s, t, g, oprm, oflt), side)


def test_more_clouds_than_one_launch_row():
    """ops.icp without ids over 70 000 problems filters 70 000 sources in one voxel stage (its per-cloud kernels take
    65 535 clouds per launch): problem p uses pair p % 8, so every result must equal its pair's oracle result."""
    base = [synth.make_icp_pair(900 + k, n_source=60, n_target=150) for k in range(8)]
    P = 70000
    pairs = [(base[p % 8][0], base[p % 8][1], base[p % 8][2].astype(F32)) for p in range(P)]
    flt, oflt = _filters(dict(reading=[(VOX, 1, 0.3)]))
    prm, oprm = _params(0)
    srcs, tgts, gs = zip(*pairs)
    sp, so = _pack(srcs)
    tp, to = _pack(tgts)
    r = ops.icp(sp, so, tp, to, torch.from_numpy(np.stack(gs)).cuda(), 60, 150, prm, filters=flt)
    got = {k: v.cpu().numpy() for k, v in r.items()}
    want = [vfr.icp(s, t, g.astype(F32), oprm, oflt) for s, t, g in base]
    for p in range(P):
        w = want[p % 8]
        assert (int(got["status"][p]), int(got["iterations"][p]), int(got["inliers"][p])) == \
            (w["status"], w["iterations"], w["inliers"]), p
        assert got["T"][p].tobytes() == np.asarray(w["T"], F32).tobytes(), p
