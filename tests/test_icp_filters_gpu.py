"""GPU: the ICP filters (sfe_icp_filters: distance data filters, MinDist / MedianDist outlier filters) bit for bit
against oracle/icp_filters_ref.c -- status, iterations, inliers and the bits of T -- through every entry point:
sfe_icp_dev on pipeline-sized pairs (one-pass search) and config-3 pairs (pruned search), the map class, the front
end's size classes (sfe_frontend_icp_dev), the batched front end against the oracle chain, the host flavours, and a
context whose filters are cleared again."""
import numpy as np
import pytest
import torch

from oracle import icp_filters_ref as fr
from oracle import oracle as orc
from sonar_slam_b200 import _lib, ops, synth
from sonar_slam_b200.bruce_slam import pcl

pytestmark = pytest.mark.gpu
F32 = np.float32
MX, MN = _lib.MAX_DIST, _lib.MIN_DIST

# name -> (trim ratio, IcpFilters keyword arguments)
SETTINGS = {
    "median": (-1.0, dict(median_factor=3.0)),
    "median_trim03": (0.3, dict(median_factor=0.75)),
    "median_trim08": (0.8, dict(median_factor=2.0)),
    "mindist": (0.8, dict(min_dist=0.02)),
    "reading_radial": (0.8, dict(reading=[(MX, -1, 18.0)])),
    "reference_axis": (0.8, dict(reference=[(MN, 0, -8.0), (MX, 1, 12.0)])),
    "all": (0.8, dict(min_dist=0.01, median_factor=1.5, reading=[(MN, -1, 1.0), (MX, 1, 15.0)],
                      reference=[(MX, -1, 25.0)])),
}


def _filters(name):
    trim, kw = SETTINGS[name]
    return trim, _lib.IcpFilters(**kw), fr.IcpFilters(**kw)


def _params(trim, minimizer):
    kw = dict(trim_ratio=trim, minimizer=minimizer, normals_knn=5)
    return _lib.IcpParams(**kw), orc.IcpParams(**kw)


def _same(got, want, what):
    assert (int(got["status"]), int(got["iterations"]), int(got["inliers"])) == \
        (want["status"], want["iterations"], want["inliers"]), what
    assert np.array_equal(np.asarray(got["T"], F32).view(np.uint32), np.asarray(want["T"], F32).view(np.uint32)), what


def _pack(clouds):
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    return torch.from_numpy(np.concatenate(clouds).astype(F32)).cuda(), torch.from_numpy(off).cuda()


def _run_dev(pairs, prm, flt, ctx=None):
    srcs, tgts, gs = zip(*pairs)
    sp, so = _pack(srcs)
    tp, to = _pack(tgts)
    g = torch.from_numpy(np.stack(gs).astype(F32)).cuda()
    r = ops.icp(sp, so, tp, to, g, max(map(len, srcs)), max(map(len, tgts)), prm, ctx=ctx, filters=flt)
    torch.cuda.synchronize()
    return [dict(T=r["T"][k].cpu().numpy(), iterations=r["iterations"][k].item(), inliers=r["inliers"][k].item(),
                 status=r["status"][k].item()) for k in range(len(pairs))]


def _pairs(kind, n=3):
    size = dict(pipeline=(400, 1400), config3=(2000, 20000))[kind]
    out = []
    for seed in range(n):
        s, t, T = synth.make_icp_pair(100 + seed, n_source=size[0], n_target=size[1])
        out.append((s, t, T.astype(F32)))
    return out


@pytest.mark.parametrize("name", list(SETTINGS))
@pytest.mark.parametrize("minimizer", [0, 1])
@pytest.mark.parametrize("kind", ["pipeline", "config3"])
def test_icp_dev_equals_oracle(kind, minimizer, name):
    trim, flt, oflt = _filters(name)
    prm, oprm = _params(trim, minimizer)
    pairs = _pairs(kind)
    got = _run_dev(pairs, prm, flt)
    for k, (s, t, g) in enumerate(pairs):
        _same(got[k], fr.icp(s, t, g, oprm, oflt), (kind, minimizer, name, k))


@pytest.mark.parametrize("name", ["median_trim03", "all"])
@pytest.mark.parametrize("minimizer", [0, 1])
def test_map_class_equals_oracle(minimizer, name):
    """A target above the in-CTA limit (map class, map_build over the compacted target), several guesses on it."""
    trim, flt, oflt = _filters(name)
    prm, oprm = _params(trim, minimizer)
    s, t, T = synth.make_icp_pair(7, n_source=1500, n_target=60000, extent=120.0)
    assert len(t) > 25000
    rng = np.random.default_rng(0)
    guesses = []
    for k in range(3):
        d = np.eye(3)
        d[:2, 2] = rng.normal(0, 0.2, 2)
        guesses.append((T @ d).astype(F32))
    icp = pcl.ICP()
    icp.params = _lib.IcpConfig(trim_ratio=trim, minimizer=minimizer, normals_knn=5, filters=flt)
    res = icp.compute_batch(s, t, guesses)
    for k, g in enumerate(guesses):
        got = dict(T=res["T"][k], iterations=res["iterations"][k], inliers=res["inliers"][k], status=res["status"][k])
        _same(got, fr.icp(s, t, g, oprm, oflt), (minimizer, name, k))


@pytest.mark.parametrize("minimizer", [0, 1])
def test_frontend_classes_equal_oracle(minimizer):
    """sfe_frontend_icp_dev: problems of several sizes go through the front end's size classes, every class used."""
    trim, flt, oflt = _filters("all")
    prm, oprm = _params(trim, minimizer)
    sizes = [(300, 600), (500, 780), (900, 2500), (350, 3000), (1500, 6000), (200, 500)]
    pairs = []
    for k, (ns, nt) in enumerate(sizes):
        s, t, T = synth.make_icp_pair(200 + k, n_source=ns, n_target=nt, extent=30.0)
        pairs.append((s, t, T.astype(F32)))
    srcs, tgts, gs = zip(*pairs)
    sp, so = _pack(srcs)
    tp, to = _pack(tgts)
    g = torch.from_numpy(np.stack(gs)).cuda()
    P = len(pairs)
    T = torch.empty((P, 3, 3), dtype=torch.float32, device="cuda")
    it, inl, st = (torch.empty(P, dtype=torch.int32, device="cuda") for _ in range(3))
    cls = torch.full((2 * P,), -1, dtype=torch.int32, device="cuda")
    ctx = ops.context(0)
    _lib.set_icp_filters(ctx, flt)
    dp = lambda x: x.data_ptr()  # noqa: E731
    import ctypes
    _lib.check(ctx.lib.sfe_frontend_icp_dev(ctx.handle, ctypes.byref(prm), dp(sp), dp(so), dp(tp), dp(to), P,
                                            max(map(len, srcs)), max(map(len, tgts)), dp(g), dp(T), dp(it), dp(inl),
                                            dp(st), dp(cls)), "sfe_frontend_icp_dev")
    _lib.set_icp_filters(ctx, None)
    torch.cuda.synchronize()
    used = set(cls[:P].cpu().tolist())
    assert used == {0, 1}, used  # the small class and the capacity class
    for k, (s, t, gg) in enumerate(pairs):
        got = dict(T=T[k].cpu().numpy(), iterations=it[k].item(), inliers=inl[k].item(), status=st[k].item())
        _same(got, fr.icp(s, t, gg, oprm, oflt), (minimizer, k))


def test_frontend_run_equals_oracle_chain(monkeypatch):
    """FrontEnd(icp_filters=...): frame clouds as readings, window submaps as references, against the oracle chain."""
    from oracle import featx_ref, pipeline_ref
    from sonar_slam_b200 import pipeline
    trim, flt, oflt = _filters("all")
    d = synth.make_trajectory_frames(10, seed=3)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    ctx = ops.context(0)
    maps = _lib.Maps(ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    fe = pipeline.FrontEnd(ctx, maps, max_frames=16, min_points=30, icp=_lib.IcpConfig(filters=flt))
    res = fe.run_host(frames, poses)
    monkeypatch.setattr(pipeline_ref.orc, "icp", lambda s, t, g, p: fr.icp(s, t, g, p, oflt))
    _, want = pipeline_ref.run(frames, poses, geo, min_points=30)
    ok = 0
    for i, w in enumerate(want):
        assert res["status"][i] == w["status"], i
        if w["status"] == 0:
            ok += 1
            got = dict(T=res["T"][i], iterations=res["iterations"][i], inliers=res["inliers"][i], status=0)
            _same(got, w, i)
    assert ok >= 5


def test_pairs_batch_equals_sequential_calls():
    """compute_pairs (one launch, data filters once per cloud) against one compute_batch call per pair."""
    trim, flt, _ = _filters("all")
    icp = pcl.ICP()
    icp.params = _lib.IcpConfig(trim_ratio=trim, filters=flt)
    pairs = _pairs("pipeline", 4)
    shift = np.array([[1, 0, 0.2], [0, 1, -0.1], [0, 0, 1]], F32)
    gs = [[g, (g @ shift).astype(F32)] for _, _, g in pairs]
    batch = icp.compute_pairs([p[0] for p in pairs], [p[1] for p in pairs], gs)
    for k, (s, t, _) in enumerate(pairs):
        one = icp.compute_batch(s, t, gs[k])
        for f in ("T", "iterations", "inliers", "status"):
            assert np.array_equal(np.asarray(batch[k][f]), np.asarray(one[f])), (k, f)


def test_cleared_filters_give_a_fresh_context():
    pairs = _pairs("pipeline", 2)
    prm = _lib.IcpParams()
    ctx = _lib.Context(0)
    fresh = _run_dev(pairs, prm, None, ctx=_lib.Context(0))
    _trim, flt, _ = _filters("all")
    filtered = _run_dev(pairs, prm, flt, ctx=ctx)
    again = _run_dev(pairs, prm, None, ctx=ctx)
    for k, (s, t, g) in enumerate(pairs):
        _same(again[k], fresh[k], k)
        _same(fresh[k], orc.icp(s, t, g, orc.IcpParams()), k)
    assert any(a["inliers"] != b["inliers"] for a, b in zip(filtered, fresh))


def test_targets_emptied_by_the_filters_raise_as_empty_targets():
    s, t, T = synth.make_icp_pair(5, n_source=300, n_target=900)
    icp = pcl.ICP()
    icp.params = _lib.IcpConfig(filters=_lib.IcpFilters(reference=[(MX, -1, 0.0)]))
    with pytest.raises(RuntimeError, match="reference cloud is empty"):
        icp.compute(s, t, T.astype(F32))
    icp.params = _lib.IcpConfig(filters=_lib.IcpFilters(reading=[(MX, -1, 0.0)]))
    assert icp.compute(s, t, T.astype(F32))[0] == "no outlier to filter"
