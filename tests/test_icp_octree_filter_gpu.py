"""GPU: OctreeGridDataPointsFilter in the ICP data-filter chains, bit for bit against oracle/octree_filter_ref.c --
status, iterations, inliers and all nine entries of T:

  * every sampler (first point, centroid, medoid) on either cloud, alone and mixed with distance filters, for
    point-to-point and point-to-plane, with the shipped checkers and with a fixed 20 iterations, on pipeline-sized
    pairs (one-CTA down-sample) and config-3 pairs (targets above the one-CTA down-sample limit: the grid-wide path);
  * one compute_pairs call whose targets take the in-CTA and the map class and whose sources take the global-source
    class, the sources also above the one-CTA down-sample limit;
  * ops.icp with and without cloud ids, and the batched front end against the oracle chain frame by frame;
  * clouds the filters leave with one point or empty.
"""
import numpy as np
import pytest
import torch

from oracle import octree_filter_ref as ofr
from oracle import oracle as orc
from sonar_slam_b200 import _lib, ops, synth
from sonar_slam_b200.bruce_slam import pcl

pytestmark = pytest.mark.gpu
F32 = np.float32
MX, MN, OCT = _lib.MAX_DIST, _lib.MIN_DIST, _lib.OCTREE

CHAINS = {
    "reading_first": dict(reading=[(OCT, 0, 0.3)]),
    "reading_centroid_mixed": dict(reading=[(MX, -1, 18.0), (OCT, 2, 0.25)]),
    "reading_medoid": dict(reading=[(OCT, 3, 0.2)]),
    "reference_first_mixed": dict(reference=[(OCT, 0, 0.15), (MN, 0, -8.0), (OCT, 2, 0.4)]),
    "reference_centroid": dict(reference=[(OCT, 2, 0.2)]),
    "reference_medoid_mixed": dict(reference=[(MX, -1, 25.0), (OCT, 3, 0.3)]),
    "both": dict(min_dist=0.01, reading=[(OCT, 3, 0.2), (MX, 1, 15.0)], reference=[(MX, -1, 25.0), (OCT, 2, 0.2)]),
}
CHECKERS = {"shipped": {}, "fixed20": dict(max_iterations=20, smooth_length=0)}


def _filters(kw):
    return _lib.IcpFilters(**kw), ofr.IcpFilters(**kw)


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


def _run_dev(pairs, prm, flt):
    srcs, tgts, gs = zip(*pairs)
    sp, so = _pack(srcs)
    tp, to = _pack(tgts)
    g = torch.from_numpy(np.stack(gs).astype(F32)).cuda()
    r = ops.icp(sp, so, tp, to, g, max(map(len, srcs)), max(map(len, tgts)), prm, filters=flt)
    torch.cuda.synchronize()
    return _rows(r, len(pairs))


def _pairs(kind, n=3):
    size = dict(pipeline=(400, 1400), config3=(2000, 20000))[kind]
    out = []
    for seed in range(n):
        s, t, T = synth.make_icp_pair(300 + seed, n_source=size[0], n_target=size[1])
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
    if kind == "config3":  # the targets are above the one-CTA down-sample limit: the grid-wide path
        assert min(len(t) for _, t, _ in pairs) > 13880
    got = _run_dev(pairs, prm, flt)
    for k, (s, t, g) in enumerate(pairs):
        want = ofr.icp(s, t, g, oprm, oflt)
        _same(got[k], want, (kind, minimizer, chain, checkers, k))
        if checkers == "fixed20" and want["status"] == 0:
            assert want["iterations"] == 20


@pytest.mark.parametrize("minimizer", [0, 1])
def test_pairs_across_launch_classes_equal_oracle(minimizer):
    """One compute_pairs call: targets of the in-CTA and the map class, sources of the shared-memory and the
    global-source class; the large sources and target are above the one-CTA down-sample limit."""
    small_s, small_t, T0 = synth.make_icp_pair(41, n_source=1500, n_target=6000, extent=40.0)
    big_s, big_t, T1 = synth.make_icp_pair(42, n_source=16000, n_target=60000, extent=120.0)
    assert len(big_t) > 25000 and len(big_s) > max(13880, ops.icp_source_limit(2, _params(minimizer)[0]))
    kw = dict(reading=[(OCT, 2, 0.1), (MX, -1, 40.0)], reference=[(OCT, 3, 0.12)])
    flt, oflt = _filters(kw)
    prm, oprm = _params(minimizer, trim_ratio=0.8)
    icp = pcl.ICP()
    icp.params = _lib.IcpConfig(trim_ratio=0.8, minimizer=minimizer, normals_knn=5, filters=flt)
    shift = np.array([[1, 0, 0.15], [0, 1, -0.1], [0, 0, 1]], F32)
    srcs, tgts = [small_s, small_s, big_s, big_s], [small_t, big_t, small_t, big_t]
    gs = [[T0.astype(F32)], [T1.astype(F32), (T1 @ shift).astype(F32)], [T0.astype(F32)], [T1.astype(F32)]]
    res = icp.compute_pairs(srcs, tgts, gs)
    ok = 0
    for k in range(4):
        for j, g in enumerate(gs[k]):
            got = dict(T=res[k]["T"][j], iterations=res[k]["iterations"][j], inliers=res[k]["inliers"][j],
                       status=res[k]["status"][j])
            want = ofr.icp(srcs[k], tgts[k], g, oprm, oflt)
            _same(got, want, (minimizer, k, j))
            ok += want["status"] == 0
    assert ok >= 2


@pytest.mark.parametrize("ids", [False, True])
def test_ops_icp_with_and_without_ids_equals_oracle(ids):
    flt, oflt = _filters(CHAINS["both"])
    prm, oprm = _params(0)
    pairs = _pairs("pipeline", 2)
    srcs, tgts = [p[0] for p in pairs], [p[1] for p in pairs]
    shift = np.array([[1, 0, 0.1], [0, 1, 0.05], [0, 0, 1]], F32)
    if ids:  # four problems over two sources and two targets, crossed
        sid, tid = [0, 1, 0, 1], [0, 1, 1, 0]
    else:
        sid, tid = [0, 1], [0, 1]
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
        _same(got[k], ofr.icp(srcs[sid[k]], tgts[tid[k]], gs[k], oprm, oflt), (ids, k))


def test_frontend_run_equals_oracle_chain(monkeypatch):
    """FrontEnd(icp_filters=...) with octree filters: frame clouds as readings, window submaps as references."""
    from oracle import featx_ref, pipeline_ref
    from sonar_slam_b200 import pipeline
    flt, oflt = _filters(dict(reading=[(OCT, 0, 0.4)], reference=[(MX, -1, 30.0), (OCT, 2, 0.3)]))
    d = synth.make_trajectory_frames(10, seed=3)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    ctx = ops.context(0)
    maps = _lib.Maps(ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    fe = pipeline.FrontEnd(ctx, maps, max_frames=16, min_points=30, icp=_lib.IcpConfig(filters=flt))
    res = fe.run_host(frames, poses)
    monkeypatch.setattr(pipeline_ref.orc, "icp", lambda s, t, g, p: ofr.icp(s, t, g, p, oflt))
    _, want = pipeline_ref.run(frames, poses, geo, min_points=30)
    ok = 0
    for i, w in enumerate(want):
        assert res["status"][i] == w["status"], i
        if w["status"] == 0:
            ok += 1
            got = dict(T=res["T"][i], iterations=res["iterations"][i], inliers=res["inliers"][i], status=0)
            _same(got, w, i)
    assert ok >= 5


@pytest.mark.parametrize("case", ["one_source_point", "one_target_point", "empty_source", "empty_target"])
def test_clouds_left_with_one_point_or_none(case):
    """An octree larger than the cloud leaves one point; a distance filter before it can leave none.  The statuses
    are the documented ones: an emptied target is SFE_ICP_EMPTY_REF, an emptied source "no outlier to filter"."""
    kw = dict(one_source_point=dict(reading=[(OCT, 2, 1e4)]),
              one_target_point=dict(reference=[(OCT, 0, 1e4)]),
              empty_source=dict(reading=[(MX, -1, 0.0), (OCT, 3, 0.2)]),
              empty_target=dict(reference=[(MX, -1, 0.0), (OCT, 2, 0.2)]))[case]
    flt, oflt = _filters(kw)
    prm, oprm = _params(0)
    pairs = _pairs("pipeline", 2)
    got = _run_dev(pairs, prm, flt)
    for k, (s, t, g) in enumerate(pairs):
        want = ofr.icp(s, t, g, oprm, oflt)
        _same(got[k], want, (case, k))
        if case == "empty_target":
            assert want["status"] == 6
        if case == "empty_source":
            assert want["status"] == 1
