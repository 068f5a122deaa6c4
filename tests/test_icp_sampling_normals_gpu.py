"""GPU: SamplingSurfaceNormalDataPointsFilter as the last reference filter of an ICP call, bit for bit against
oracle/sampling_normal_ref.c -- status, iterations, inliers and all nine entries of T:

  * point-to-plane reading the filter's normals and point-to-point with the filter as a down-sampler, samplingMethod 0
    (ratio 1) and 1, knn 3, 7 and 64, shipped and fixed-iteration checkers;
  * behind MaxDist, octree and voxel filters, and with a RobustOutlierFilter;
  * the in-CTA class and the map class (a 243 k-point map target) in one call, through ops.icp, compute_batch (ids)
    and compute_pairs, and an icp.yaml through ICP.compute;
  * a target the filter empties (every box above maxBoxDim) and an empty target.
"""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import robust_ref
from oracle import sampling_normal_ref as snr
from sonar_slam_b200 import _lib, ops, synth
from sonar_slam_b200.bruce_slam import pcl

pytestmark = pytest.mark.gpu
F32 = np.float32
MX, OCT, VOX, SN = _lib.MAX_DIST, _lib.OCTREE, _lib.VOXEL, _lib.SAMPLING_NORMALS
CHECKERS = {"shipped": {}, "fixed20": dict(max_iterations=20, smooth_length=0)}


def _params(minimizer, knn, **kw):
    kw = dict(minimizer=minimizer, normals_knn=knn, **kw)
    return _lib.IcpParams(**kw), orc.IcpParams(**kw)


def _filters(**kw):
    return _lib.IcpFilters(**kw), snr.IcpFilters(**kw)


def _same(got, want, what):
    assert (int(got["status"]), int(got["iterations"]), int(got["inliers"])) == \
        (want["status"], want["iterations"], want["inliers"]), what
    assert np.array_equal(np.asarray(got["T"], F32).view(np.uint32), np.asarray(want["T"], F32).view(np.uint32)), what


def _pack(clouds):
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    return torch.from_numpy(np.concatenate(clouds).astype(F32)).cuda(), torch.from_numpy(off).cuda()


def _run_dev(pairs, prm, flt, robust=None):
    srcs, tgts, gs = zip(*pairs)
    sp, so = _pack(srcs)
    tp, to = _pack(tgts)
    g = torch.from_numpy(np.stack(gs).astype(F32)).cuda()
    r = ops.icp(sp, so, tp, to, g, max(map(len, srcs)), max(map(len, tgts)), prm, filters=flt, robust=robust)
    torch.cuda.synchronize()
    return [dict(T=r["T"][k].cpu().numpy(), iterations=r["iterations"][k].item(), inliers=r["inliers"][k].item(),
                 status=r["status"][k].item()) for k in range(len(pairs))]


def _pairs(n=3, ns=400, nt=1400, seed=500):
    out = []
    for k in range(n):
        s, t, T = synth.make_icp_pair(seed + k, n_source=ns, n_target=nt)
        out.append((s, t, T.astype(F32)))
    return out


@pytest.mark.parametrize("checkers", list(CHECKERS))
@pytest.mark.parametrize("knn", [3, 7, 64])
@pytest.mark.parametrize("method", [0, 1])
@pytest.mark.parametrize("minimizer", [0, 1])
def test_icp_dev_equals_oracle(minimizer, method, knn, checkers):
    prm, oprm = _params(minimizer, knn, **CHECKERS[checkers])
    flt, oflt = _filters(reference=[(SN, method, np.inf)])
    pairs = _pairs() + _pairs(1, 2000, 20000, seed=900)
    got = _run_dev(pairs, prm, flt)
    for k, (s, t, g) in enumerate(pairs):
        _same(got[k], snr.icp(s, t, g, oprm, oflt), (minimizer, method, knn, checkers, k))


CHAINS = {
    "maxdist": dict(reference=[(MX, -1, 25.0), (SN, 1, np.inf)]),
    "octree": dict(reference=[(OCT, 2, 0.2), (SN, 0, np.inf)]),
    "voxel": dict(reading=[(VOX, 1, 0.2)], reference=[(VOX, 1, 0.1), (SN, 1, 1.5)]),
    "outlier": dict(min_dist=0.01, median_factor=4.0, reference=[(SN, 1, np.inf)]),
}


@pytest.mark.parametrize("robust", [None, "huber", "cauchy"])
@pytest.mark.parametrize("chain", list(CHAINS))
def test_chains_and_robust(chain, robust):
    prm, oprm = _params(1, 7)
    flt, oflt = _filters(**CHAINS[chain])
    rb = _lib.IcpRobust(robust, 0.5) if robust else None
    orb = robust_ref.Robust(robust, 0.5) if robust else None
    pairs = _pairs(3, seed=600)
    got = _run_dev(pairs, prm, flt, rb)
    for k, (s, t, g) in enumerate(pairs):
        _same(got[k], snr.icp(s, t, g, oprm, oflt, orb), (chain, robust, k))


@pytest.mark.parametrize("minimizer", [0, 1])
def test_map_target_and_small_targets_in_one_call(minimizer):
    """A 243 k-point map target (the map class, the grid-wide filter level count) next to pipeline-sized problems"""
    big = synth.make_map_cloud(243_000, seed=3)[0]
    rng = np.random.default_rng(4)
    src = big[rng.choice(len(big), 3000, replace=False)] + F32(0.05)
    prm, oprm = _params(minimizer, 7)
    flt, oflt = _filters(reference=[(SN, 1, np.inf)])
    pairs = [(src.astype(F32), big.astype(F32), np.eye(3, dtype=F32))] + _pairs(2)
    got = _run_dev(pairs, prm, flt)
    for k, (s, t, g) in enumerate(pairs):
        want = snr.icp(s, t, g, oprm, oflt)
        _same(got[k], want, (minimizer, k))
    assert got[0]["status"] == 0


def test_batch_pairs_and_yaml():
    text = ("referenceDataPointsFilters:\n  - MaxDistDataPointsFilter: {maxDist: 30.0}\n"
            "  - SamplingSurfaceNormalDataPointsFilter: {knn: 9, samplingMethod: 1}\n"
            "matcher:\n  KDTreeMatcher:\n    maxDist: 10.0\noutlierFilters:\n  - TrimmedDistOutlierFilter: {ratio: 0.8}\n"
            "errorMinimizer:\n  PointToPlaneErrorMinimizer\n")
    icp = pcl.ICP()
    icp.params = pcl.parse_icp_yaml(text)
    oprm = orc.IcpParams(**{f: getattr(icp.params, f) for f, _ in _lib.IcpParams._fields_})
    oflt = snr.IcpFilters(reference=[(MX, -1, 30.0), (SN, 1, np.inf)])
    pairs = _pairs(3, seed=700)
    for s, t, g in pairs:
        msg, T = icp.compute(s, t, g)
        want = snr.icp(s, t, g, oprm, oflt)
        assert msg == want["message"] and np.array_equal(T.view(np.uint32), np.asarray(want["T"], F32).view(np.uint32))
    s, t, _ = pairs[0]
    gs = np.stack([p[2] for p in pairs])
    r = icp.compute_batch(s, t, gs)
    for k in range(len(gs)):
        want = snr.icp(s, t, gs[k], oprm, oflt)
        assert np.array_equal(r["T"][k].view(np.uint32), np.asarray(want["T"], F32).view(np.uint32))
    r = icp.compute_pairs([p[0] for p in pairs], [p[1] for p in pairs], [[p[2]] for p in pairs])
    for k, (s, t, g) in enumerate(pairs):
        want = snr.icp(s, t, g, oprm, oflt)
        assert np.array_equal(r[k]["T"][0].view(np.uint32), np.asarray(want["T"], F32).view(np.uint32))


def test_emptied_and_empty_targets():
    prm, oprm = _params(1, 7)
    flt, oflt = _filters(reference=[(SN, 1, 0.0)])  # every box of distinct points is dropped
    s, t, g = _pairs(1)[0]
    got = _run_dev([(s, t, g)], prm, flt)[0]
    want = snr.icp(s, t, g, oprm, oflt)
    _same(got, want, "emptied")
    assert want["status"] == 6
    got = _run_dev([(s, np.zeros((0, 2), F32), g), (s, t, g)], prm, _lib.IcpFilters(reference=[(SN, 1, np.inf)]))
    assert got[0]["status"] == 6
    _same(got[1], snr.icp(s, t, g, oprm, snr.IcpFilters(reference=[(SN, 1, np.inf)])), "next to an empty target")


# ---------------------------------------------------------------- the stage alone, the other launch classes
def _stage(clouds, knn, method, max_box, ctx=None):
    import ctypes
    ctx = ctx or ops.context(0)
    n_max = max(1, max(len(c) for c in clouds))
    pts, off = _pack([np.asarray(c, F32).reshape(-1, 2) for c in clouds])
    out = torch.empty((len(clouds) * n_max, 2), dtype=torch.float32, device="cuda")
    nrm = torch.empty_like(out)
    cnt = torch.empty(len(clouds), dtype=torch.int32, device="cuda")
    p_ = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    _lib.check(ctx.lib.sfe_icp_sampling_normals_dev(ctx.handle, p_(pts), p_(off), len(clouds), n_max, knn, method,
                                                    float(max_box), p_(out), p_(nrm), p_(cnt)),
               "sfe_icp_sampling_normals_dev")
    torch.cuda.synchronize()
    out, nrm, cnt = out.cpu().numpy(), nrm.cpu().numpy(), cnt.cpu().numpy()
    return [(out[c * n_max:c * n_max + cnt[c]], nrm[c * n_max:c * n_max + cnt[c]]) for c in range(len(clouds))]


def _stage_same(got, clouds, knn, method, max_box, what):
    for c, (pts, (gp, gn)) in enumerate(zip(clouds, got)):
        wp, wn = snr.sampling_normals(pts, knn, method, max_box)
        assert gp.shape == wp.shape, (what, c, len(pts))
        assert np.array_equal(gp.view(np.uint32), wp.view(np.uint32)), (what, c, len(pts))
        assert np.array_equal(gn.view(np.uint32), wn.view(np.uint32)), (what, c, len(pts))


def _stage_clouds():
    rng = np.random.default_rng(11)
    lattice = (np.stack(np.meshgrid(np.arange(70), np.arange(60)), -1).reshape(-1, 2) * 0.1).astype(F32)
    lattice = np.concatenate([lattice, lattice[:500], -lattice[:300]])[rng.permutation(len(lattice) + 800)]
    return [np.zeros((0, 2), F32), np.array([[1.0, 2.0]], F32), rng.normal(0, 2, (3, 2)).astype(F32),
            np.tile(np.array([[0.5, -0.5]], F32), (40, 1)), lattice[:4095], lattice[:4096], lattice[:4097],
            synth.make_icp_pair(5, n_source=100, n_target=9000)[1]]


@pytest.mark.parametrize("max_box", [np.inf, 0.3])
@pytest.mark.parametrize("method", [0, 1])
@pytest.mark.parametrize("knn", [3, 7, 64])
def test_stage_equals_oracle_around_the_one_cta_limit(knn, method, max_box):
    """Clouds of 0, 1, 3 and 40 coincident points, lattice clouds with ties of 4095 / 4096 (one CTA each) and 4097
    points, and 9 000 points (the grid-wide levels), in one call"""
    clouds = _stage_clouds()
    _stage_same(_stage(clouds, knn, method, max_box), clouds, knn, method, max_box, (knn, method, max_box))


@pytest.mark.parametrize("knn", [3, 7])
def test_stage_on_a_map_cloud(knn):
    big = synth.make_map_cloud(243_000, seed=3)[0]
    clouds = [big, big[:2000]]
    _stage_same(_stage(clouds, knn, 1, np.inf), clouds, knn, 1, np.inf, knn)


def test_stage_and_icp_past_one_wave():
    """A context capped at one SM: the one-CTA stage and the in-CTA ICP launch take many work items per CTA"""
    ctx = ops.context(0)
    ctx.set_grid_sms(1)
    try:
        clouds = [synth.make_icp_pair(40 + k, n_source=10, n_target=300 + 37 * k)[1] for k in range(40)]
        _stage_same(_stage(clouds, 7, 1, np.inf, ctx), clouds, 7, 1, np.inf, "one SM")
        prm, oprm = _params(1, 7)
        flt, oflt = _filters(reference=[(SN, 1, np.inf)])
        pairs = [(s, t, g) for s, t, g in _pairs(24, 300, 900, seed=800)]
        srcs, tgts, gs = zip(*pairs)
        sp, so = _pack(srcs)
        tp, to = _pack(tgts)
        g = torch.from_numpy(np.stack(gs)).cuda()
        r = ops.icp(sp, so, tp, to, g, max(map(len, srcs)), max(map(len, tgts)), prm, filters=flt, ctx=ctx)
        torch.cuda.synchronize()
        for k, (s, t, gg) in enumerate(pairs):
            got = dict(T=r["T"][k].cpu().numpy(), iterations=r["iterations"][k].item(), inliers=r["inliers"][k].item(),
                       status=r["status"][k].item())
            _same(got, snr.icp(s, t, gg, oprm, oflt), ("one SM", k))
    finally:
        ctx.set_grid_sms(0)


def test_global_source_class():
    """A source above the shared-memory layouts' limit: the global-source class, normals gathered by map_build"""
    prm, oprm = _params(1, 7)
    flt, oflt = _filters(reference=[(SN, 1, np.inf)])
    S = ops.icp_source_limit(2, prm, flt)
    pairs = [(s, t, g) for s, t, g in _pairs(1, S + 300, 20000, seed=950)] + _pairs(1)
    got = _run_dev(pairs, prm, flt)
    for k, (s, t, g) in enumerate(pairs):
        _same(got[k], snr.icp(s, t, g, oprm, oflt), ("gsrc", k))
    assert got[0]["status"] == 0


def test_ops_icp_with_ids():
    prm, oprm = _params(1, 7)
    flt, oflt = _filters(reference=[(MX, -1, 28.0), (SN, 0, np.inf)])
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
        _same(got, snr.icp(srcs[sid[k]], tgts[tid[k]], gs[k], oprm, oflt), ("ids", k))


@pytest.mark.parametrize("minimizer", [0, 1])
def test_frontend_size_classes_equal_oracle(minimizer):
    """sfe_frontend_icp_dev: frame-sized problems in the narrow / small class (the dense 64-register instantiations)
    and above it, the filter set on the context"""
    import ctypes
    sizes = [(300, 420), (500, 700), (900, 1200), (1400, 2500)]
    prm, oprm = _params(minimizer, 7)
    flt, oflt = _filters(reference=[(MX, -1, 30.0), (SN, 1, np.inf)])
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
        want = snr.icp(s, t, g, oprm, oflt)
        _same(got, want, (minimizer, k))
        ok += want["status"] == 0
    assert ok >= 2


def test_frontend_run_equals_oracle_chain(monkeypatch):
    """FrontEnd(icp=IcpConfig(filters=...)) with the filter down-sampling the window submaps, frame for frame against
    oracle/pipeline_ref"""
    from oracle import featx_ref, pipeline_ref
    from sonar_slam_b200 import pipeline
    flt, oflt = _filters(reference=[(MX, -1, 30.0), (SN, 1, np.inf)])
    d = synth.make_trajectory_frames(10, seed=3)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    ctx = ops.context(0)
    maps = _lib.Maps(ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    fe = pipeline.FrontEnd(ctx, maps, max_frames=16, min_points=30, icp=_lib.IcpConfig(filters=flt))
    res = fe.run_host(frames, poses)
    monkeypatch.setattr(pipeline_ref.orc, "icp", lambda s, t, g, p: snr.icp(s, t, g, p, oflt))
    _, want = pipeline_ref.run(frames, poses, geo, min_points=30)
    ok = 0
    for i, w in enumerate(want):
        assert res["status"][i] == w["status"], i
        if w["status"] == 0:
            ok += 1
            _same(dict(T=res["T"][i], iterations=res["iterations"][i], inliers=res["inliers"][i], status=0), w, i)
    assert ok >= 5
