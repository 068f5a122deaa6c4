"""GPU: the RobustOutlierFilter in the 2-D scan matcher, bit for bit against oracle/robust_ref.c -- status, iterations,
inliers and all nine entries of T:

  * every robustFct, point-to-point and point-to-plane, with a fixed 20 iterations and with the shipped checkers, on
    config-3 pairs (2 000 x 20 000 points: 200 pairs point-to-point; 6 point-to-plane, whose oracle computes the
    normals by brute force);
  * combined with MaxDist / Trimmed / MinDist / Median and a data filter, and with the approximation cut-off;
  * sources at ops.icp_source_limit and one past it (the global-source class), targets at ops.icp_cta_limit and one
    past it (the map class), through compute, compute_batch and compute_pairs;
  * the front end's size classes (sfe_frontend_icp_dev) and the batched front end against the oracle chain;
  * persistent CTAs taking many work items in a row (Context.set_grid_sms);
  * L1 at e2 == 0 (an infinite weight: NaN sums), the same pairs dropped by MinDist (inf * 0 = NaN, kept), every
    weight zero ("no point to minimize"), and 3-D clouds refused before any launch.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from oracle import robust_ref as rr
from sonar_slam_b200 import _lib, ops, synth
from sonar_slam_b200.bruce_slam import pcl

pytestmark = pytest.mark.gpu
F32 = np.float32
MX = _lib.MAX_DIST
# tunings that give every function a spread of weights on these scenes (squared distances of a few cm^2 to m^2)
TUNING = {"cauchy": 0.05, "welsch": 0.1, "sc": 0.01, "gm": 0.02, "tukey": 0.2, "huber": 0.05, "L1": 1.0}
CHECKERS = {"shipped": {}, "fixed20": dict(max_iterations=20, smooth_length=0)}


def _robust(fct, tuning=None, approximation=float("inf")):
    k = TUNING[fct] if tuning is None else tuning
    return _lib.IcpRobust(fct, k, approximation), rr.Robust(fct, k, approximation)


def _params(minimizer=0, **kw):
    kw = dict(minimizer=minimizer, normals_knn=5, **kw)
    return _lib.IcpParams(**kw), orc.IcpParams(**kw)


def _same(got, want, what):
    assert (int(got["status"]), int(got["iterations"]), int(got["inliers"])) == \
        (want["status"], want["iterations"], want["inliers"]), (what, got, want)
    assert np.array_equal(np.asarray(got["T"], F32).view(np.uint32), np.asarray(want["T"], F32).view(np.uint32)), what


def _pack(clouds):
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    return torch.from_numpy(np.concatenate(clouds).astype(F32)).cuda(), torch.from_numpy(off).cuda()


def _rows(r, P):
    return [dict(T=r["T"][k].cpu().numpy(), iterations=r["iterations"][k].item(), inliers=r["inliers"][k].item(),
                 status=r["status"][k].item()) for k in range(P)]


def _run_dev(pairs, prm, rob, flt=None, ctx=None):
    srcs, tgts, gs = zip(*pairs)
    sp, so = _pack(srcs)
    tp, to = _pack(tgts)
    g = torch.from_numpy(np.stack(gs).astype(F32)).cuda()
    r = ops.icp(sp, so, tp, to, g, max(map(len, srcs)), max(map(len, tgts)), prm, filters=flt, robust=rob, ctx=ctx)
    torch.cuda.synchronize()
    return _rows(r, len(pairs))


_CACHE = {}


def _pairs(kind, n):
    size = dict(pipeline=(400, 1400), config3=(2000, 20000))[kind]
    key = (kind, n)
    if key not in _CACHE:
        out = []
        for seed in range(n):
            s, t, T = synth.make_icp_pair(500 + seed, n_source=size[0], n_target=size[1])
            out.append((s, t, T.astype(F32)))
        _CACHE[key] = out
    return _CACHE[key]


@pytest.mark.parametrize("checkers", list(CHECKERS))
@pytest.mark.parametrize("fct", list(TUNING))
@pytest.mark.parametrize("minimizer", [0, 1])
def test_config3_equals_oracle(minimizer, fct, checkers):
    rob, orob = _robust(fct)
    prm, oprm = _params(minimizer, **CHECKERS[checkers])
    pairs = _pairs("config3", 200 if minimizer == 0 else 6)
    got = _run_dev(pairs, prm, rob)
    ok = 0
    for k, (s, t, g) in enumerate(pairs):
        want = rr.icp(s, t, g, oprm, robust=orob)
        _same(got[k], want, (minimizer, fct, checkers, k))
        ok += want["status"] == 0
    assert ok >= len(pairs) // 2


def test_huber_above_every_kept_distance_is_the_unweighted_chain():
    """Huber with k^2 above maxDist^2 weighs every kept pair 1: the ROBUST kernels give the shipped kernels' bits."""
    rob, _ = _robust("huber", 100.0)
    for minimizer in (0, 1):
        prm, _ = _params(minimizer)
        pairs = _pairs("pipeline", 4)
        got = _run_dev(pairs, prm, rob)
        base = _run_dev(pairs, prm, None)
        for k in range(len(pairs)):
            _same(got[k], base[k], (minimizer, k))


FILTERED = {
    "maxdist_trim": (dict(), dict()),
    "min_median": (dict(), dict(min_dist=0.01, median_factor=2.5)),
    "data_filter": (dict(trim_ratio=-1.0), dict(reading=[(MX, -1, 18.0)], reference=[(MX, -1, 30.0)])),
    "all": (dict(trim_ratio=0.7), dict(min_dist=0.005, median_factor=3.0, reading=[(MX, 0, 15.0)])),
}


@pytest.mark.parametrize("setting", list(FILTERED))
@pytest.mark.parametrize("fct", ["cauchy", "tukey", "L1"])
@pytest.mark.parametrize("minimizer", [0, 1])
def test_combined_with_other_filters_equals_oracle(minimizer, fct, setting):
    pkw, fkw = FILTERED[setting]
    rob, orob = _robust(fct, approximation=4.0 if setting == "all" else float("inf"))
    prm, oprm = _params(minimizer, **pkw)
    flt = _lib.IcpFilters(**fkw) if fkw else None
    oflt = rr.IcpFilters(**fkw) if fkw else None
    for kind, n in (("pipeline", 4), ("config3", 2)):
        pairs = _pairs(kind, n)
        got = _run_dev(pairs, prm, rob, flt)
        for k, (s, t, g) in enumerate(pairs):
            _same(got[k], rr.icp(s, t, g, oprm, oflt, orob), (kind, minimizer, fct, setting, k))


def _cloud(n, seed, extent=60.0):
    s, _, _ = synth.make_icp_pair(seed, n_source=n, n_target=10, extent=extent)
    return s[:n].astype(F32)


@pytest.mark.parametrize("minimizer", [0, 1])
def test_launch_classes_at_their_bounds(minimizer):
    """Sources at S = ops.icp_source_limit (with the robust filter) and S + 1, targets at L = ops.icp_cta_limit(S) and
    L + 1, through compute, compute_batch and compute_pairs (one call over every class)."""
    rob, orob = _robust("cauchy")
    prm, oprm = _params(minimizer)
    S = ops.icp_source_limit(2, prm, robust=rob)
    L = ops.icp_cta_limit(2, S)
    if minimizer == 0:  # the point-to-point layout does not grow with the robust filter
        assert S == ops.icp_source_limit(2, prm)
    else:  # point-to-plane: seq_sum9_warp's scratch moves off the distances
        assert S < ops.icp_source_limit(2, prm)
    base_s, base_t, T = synth.make_icp_pair(31, n_source=S + 1, n_target=L + 1, extent=80.0)
    srcs = [base_s[:S].astype(F32), base_s[:S + 1].astype(F32)]
    tgts = [base_t[:L].astype(F32), base_t[:L + 1].astype(F32)]
    icp = pcl.ICP()
    icp.params = _lib.IcpConfig(minimizer=minimizer, normals_knn=5, robust=rob)
    gs = [T.astype(F32), (T @ np.array([[1, 0, 0.1], [0, 1, -0.05], [0, 0, 1]], F32)).astype(F32)]
    want = {(i, j, k): rr.icp(s, t, g, oprm, robust=orob)
            for i, s in enumerate(srcs) for j, t in enumerate(tgts) for k, g in enumerate(gs)}
    msg, Tg = icp.compute(srcs[1], tgts[1], gs[0])
    assert msg == want[1, 1, 0]["message"] and np.array_equal(Tg.view(np.uint32), want[1, 1, 0]["T"].view(np.uint32))
    res = icp.compute_batch(srcs[0], tgts[1], gs)
    for k in range(len(gs)):
        got = dict(T=res["T"][k], iterations=res["iterations"][k], inliers=res["inliers"][k], status=res["status"][k])
        _same(got, want[0, 1, k], ("batch", k))
    pairs = [(i, j) for i in range(2) for j in range(2)]
    res = icp.compute_pairs([srcs[i] for i, _ in pairs], [tgts[j] for _, j in pairs], [gs] * len(pairs))
    for p, (i, j) in enumerate(pairs):
        for k in range(len(gs)):
            got = dict(T=res[p]["T"][k], iterations=res[p]["iterations"][k], inliers=res[p]["inliers"][k],
                       status=res[p]["status"][k])
            _same(got, want[i, j, k], ("pairs", i, j, k))


@pytest.mark.parametrize("minimizer", [0, 1])
def test_frontend_size_classes_equal_oracle(minimizer):
    """sfe_frontend_icp_dev: frame-sized problems in the narrow / small class and above it, the robust filter set on
    the context."""
    sizes = [(300, 420), (500, 700), (640, 800), (641, 801), (900, 1200), (1400, 2500)]
    rob, orob = _robust("welsch")
    prm, oprm = _params(minimizer)
    probs = []
    for k, (ns, nt) in enumerate(sizes):
        s, t, T = synth.make_icp_pair(60 + k, n_source=ns, n_target=nt)
        probs.append((s[:ns], t[:nt], T.astype(F32)))
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
    _lib.set_icp_robust(ctx, rob)
    p_ = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    try:
        _lib.check(ctx.lib.sfe_frontend_icp_dev(ctx.handle, ctypes.byref(prm), p_(src), p_(soff), p_(tgt), p_(toff), P,
                                                max(len(p[0]) for p in probs), max(len(p[1]) for p in probs),
                                                p_(guess), p_(T), p_(iters), p_(inl), p_(st), None),
                   "sfe_frontend_icp_dev")
        torch.cuda.synchronize()
    finally:
        _lib.set_icp_robust(ctx, None)
    for k, (s, t, g) in enumerate(probs):
        got = dict(T=T[k].cpu().numpy(), iterations=iters[k].item(), inliers=inl[k].item(), status=st[k].item())
        _same(got, rr.icp(s, t, g, oprm, robust=orob), (minimizer, k))


def test_frontend_run_equals_oracle_chain(monkeypatch):
    """FrontEnd(icp=IcpConfig(robust=...)): frame clouds as readings, window submaps as references, frame for frame
    against oracle/pipeline_ref with the robust chain."""
    from oracle import featx_ref, pipeline_ref
    from sonar_slam_b200 import pipeline
    rob, orob = _robust("cauchy", 0.3)
    d = synth.make_trajectory_frames(10, seed=3)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    ctx = ops.context(0)
    maps = _lib.Maps(ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    fe = pipeline.FrontEnd(ctx, maps, max_frames=16, min_points=30, icp=_lib.IcpConfig(robust=rob))
    res = fe.run_host(frames, poses)
    monkeypatch.setattr(pipeline_ref.orc, "icp", lambda s, t, g, p: rr.icp(s, t, g, p, robust=orob))
    _, want = pipeline_ref.run(frames, poses, geo, min_points=30)
    ok = 0
    for i, w in enumerate(want):
        assert res["status"][i] == w["status"], i
        if w["status"] == 0:
            ok += 1
            got = dict(T=res["T"][i], iterations=res["iterations"][i], inliers=res["inliers"][i], status=0)
            _same(got, w, i)
    assert ok >= 5


def test_persistent_ctas_take_many_items():
    """One SM's worth of persistent CTAs (Context.set_grid_sms(1)): each CTA solves many problems in a row, with the
    weights of one problem parked in dist[] before the next problem's search."""
    ctx = _lib.Context(0, torch.cuda.current_stream(0).cuda_stream)
    try:
        assert ctx.set_grid_sms(1) == 1
        pairs = _pairs("pipeline", 4) * 6
        for minimizer in (0, 1):
            rob, orob = _robust("gm")
            prm, oprm = _params(minimizer)
            got = _run_dev(pairs, prm, rob, ctx=ctx)
            for k, (s, t, g) in enumerate(pairs):
                _same(got[k], rr.icp(s, t, g, oprm, robust=orob), (minimizer, k))
    finally:
        ctx.close()


@pytest.mark.parametrize("checkers", ["shipped", "fixed20", "smooth1"])
@pytest.mark.parametrize("min_dist", [None, 0.01])
def test_l1_at_zero_distance(min_dist, checkers):
    """Source == target and the identity guess: every e2 is 0, so L1's weight is inf and the sums NaN.  MinDist then
    drops every pair, and inf * 0 = NaN keeps them all.  A differential checker that looks back one step reports a NaN
    point-to-point fit (status 3 / 4); the shipped one (smoothLength 4) has not looked yet when the next iteration's NaN
    points find no match ("no outlier to filter")."""
    s, t, _ = _pairs("pipeline", 1)[0]
    rob, orob = _robust("L1")
    prm, oprm = _params(0, **dict(CHECKERS, smooth1=dict(smooth_length=1))[checkers])
    flt = _lib.IcpFilters(min_dist=min_dist) if min_dist is not None else None
    oflt = rr.IcpFilters(min_dist=min_dist) if min_dist is not None else None
    g = np.eye(3, dtype=F32)
    for minimizer in (0, 1):
        prm.minimizer = oprm.minimizer = minimizer
        want = rr.icp(t, t, g, oprm, oflt, orob)
        got = _run_dev([(t, t, g)], prm, rob, flt)[0]
        _same(got, want, (minimizer, min_dist, checkers))
        assert want["inliers"] == len(t) or want["iterations"] == 0
        if checkers == "smooth1" and minimizer == 0:  # (point-to-plane: NaN pivots leave every unknown 0)
            assert want["status"] in (3, 4)


@pytest.mark.parametrize("how", ["tukey", "approximation"])
def test_every_weight_zero(how):
    """Tukey with a tiny k, or an approximation of 0: no pair keeps a weight, "no point to minimize"."""
    rob, orob = _robust("tukey", 1e-6) if how == "tukey" else _robust("cauchy", approximation=0.0)
    for minimizer in (0, 1):
        prm, oprm = _params(minimizer)
        pairs = _pairs("pipeline", 2)
        got = _run_dev(pairs, prm, rob)
        for k, (s, t, g) in enumerate(pairs):
            want = rr.icp(s, t, g, oprm, robust=orob)
            assert want["status"] == 2
            _same(got[k], want, (how, minimizer, k))


def test_3d_refused_before_any_launch():
    rob, _ = _robust("cauchy")
    ctx = ops.context(0)
    s = torch.rand(50, 3, device="cuda")
    off = torch.tensor([0, 50], dtype=torch.int32, device="cuda")
    g = torch.eye(4, device="cuda")[None].contiguous()
    before = ctx.launches
    with pytest.raises(_lib.SonarFEError, match="RobustOutlierFilter"):
        ops.icp(s, off, s, off, g, 50, 50, _lib.IcpParams(), robust=rob, ctx=ctx)
    assert ctx.launches == before
    _lib.set_icp_robust(ctx, None)
    icp = pcl.ICP()
    icp.params = _lib.IcpConfig(robust=rob)
    with pytest.raises(NotImplementedError, match="RobustOutlierFilter"):
        icp.compute(np.zeros((10, 3), F32), np.zeros((10, 3), F32), np.eye(4, dtype=F32))
    assert ctx.launches == before


def test_yaml_through_the_slam_mirror():
    """pcl.ICP.loadFromYaml-style parsing of a YAML with a RobustOutlierFilter next to the shipped filters, through
    compute_pairs, against the oracle."""
    text = ("matcher:\n  KDTreeMatcher:\n    maxDist: 10.0\n"
            "outlierFilters:\n  - MaxDistOutlierFilter:\n      maxDist: 3.0\n"
            "  - RobustOutlierFilter:\n      robustFct: huber\n      tuning: 0.05\n      scaleEstimator: none\n"
            "  - TrimmedDistOutlierFilter:\n      ratio: 0.8\n"
            "errorMinimizer:\n  PointToPointErrorMinimizer\n"
            "transformationCheckers:\n  - CounterTransformationChecker:\n      maxIterationCount: 40\n"
            "  - DifferentialTransformationChecker:\n      minDiffRotErr: 0.01\n      minDiffTransErr: 0.1\n"
            "      smoothLength: 4\n")
    icp = pcl.ICP()
    icp.params = pcl.parse_icp_yaml(text)
    oprm = orc.IcpParams(**{f: getattr(icp.params, f) for f, _ in _lib.IcpParams._fields_})
    orob = rr.Robust("huber", 0.05)
    pairs = _pairs("pipeline", 3)
    res = icp.compute_pairs([p[0] for p in pairs], [p[1] for p in pairs], [[p[2]] for p in pairs])
    for k, (s, t, g) in enumerate(pairs):
        got = dict(T=res[k]["T"][0], iterations=res[k]["iterations"][0], inliers=res[k]["inliers"][0],
                   status=res[k]["status"][0])
        _same(got, rr.icp(s, t, g, oprm, robust=orob), k)
