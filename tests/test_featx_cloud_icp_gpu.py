"""GPU parity (through the C ABI) for the stages after CFAR: polar->Cartesian cloud, cloud
filters, NN match and the ICP scan matcher, against the CPU oracle and the golden fixtures."""
import numpy as np
import pytest
import torch

from oracle import featx_ref, oracle as orc
from sonar_slam_b200 import _lib, ops, synth

pytestmark = pytest.mark.gpu
TAU_SOCA = 2.749063720096473


def _geo(tag="uniform", R=512, res=30.0 / 512):
    b = synth.bearings_uniform(512) if tag == "uniform" else synth.bearings_oculus(512)
    return featx_ref.Geometry(res, R, b)


def _maps(ctx, geo, R, B):
    return _lib.Maps(ctx, geo.map_x, geo.map_y, R, B, geo.width, geo.height)


# ------------------------------------------------------------------ polar -> Cartesian
@pytest.mark.parametrize("tag", ["uniform", "oculus"])
def test_cart_points_equal_reference_callback_fixture(gpu_ctx, tag, golden_dir):
    g = np.load(f"{golden_dir}/featx_config1.npz")
    geo = _geo(tag)
    maps = _maps(gpu_ctx, geo, 512, 512)
    img = torch.from_numpy(synth.make_frame(1)).cuda()
    det = ops.cfar(img, "SOCA", 20, 5, TAU_SOCA, gate=65, want_bits=True)
    for kw in (dict(mask=det["mask"]), dict(bits=det["bits"])):
        out = ops.cart_points(maps, capacity=4096, **kw)
        k = int(out["count"][0])
        assert k == len(g[tag + "_locs"])
        assert np.array_equal(out["ij"][0, :k].cpu().numpy(), g[tag + "_locs"])
        assert np.array_equal(out["xy"][0, :k].cpu().numpy(), g[tag + "_points"].astype(np.float32))


def test_cart_points_batches_random_masks_vs_cv2(gpu_ctx):
    geo = _geo("oculus")
    maps = _maps(gpu_ctx, geo, 512, 512)
    rng = np.random.default_rng(0)
    F = 600                                                     # exercises the 4-frames-per-CTA variant
    masks = np.zeros((F, 512, 512), np.uint8)
    for f in range(F):
        masks[f] = rng.random((512, 512)) < (0.002 if f % 7 else 0.05)
    out = ops.cart_points(maps, mask=torch.from_numpy(masks).cuda(), capacity=40000)
    cnt = out["count"].cpu().numpy()
    for f in list(range(0, F, 37)) + [F - 1]:
        locs, pts = featx_ref.cart_points(masks[f], geo)
        assert cnt[f] == len(locs)
        assert np.array_equal(out["ij"][f, :cnt[f]].cpu().numpy(), locs)
        assert np.array_equal(out["xy"][f, :cnt[f]].cpu().numpy(), pts.astype(np.float32))
    small = ops.cart_points(maps, mask=torch.from_numpy(masks[:3]).cuda(), capacity=10)   # capacity overflow
    assert np.array_equal(small["count"].cpu().numpy(), cnt[:3])
    assert np.array_equal(small["ij"][1].cpu().numpy(), out["ij"][1, :10].cpu().numpy())


def _odd_geo():
    return featx_ref.Geometry(0.1, 200, np.round(np.linspace(-3000, 3500, 96)).astype(np.int16))


def _bits(masks):
    """0/1 masks [F, R, B] as a CFAR bit plane: int32 [F, R, ceil(B/32)], bit b & 31 of word b >> 5 is beam b."""
    F, R, B = masks.shape
    padded = np.zeros((F, R, (B + 31) // 32 * 32), np.uint8)
    padded[..., :B] = masks
    return torch.from_numpy(np.packbits(padded, axis=-1, bitorder="little").view("<i4")).cuda()


def test_cart_points_dense_and_detection_driven_kernels_agree(gpu_ctx):
    """Each Cartesian-points kernel against the oracle, from masks and from bit planes, on a geometry cart_points_run
    sends it to.  The detection-driven scatter kernel needs the rank table of Cartesian word pairs to fit in the polar
    plane, (cw + 1) / 2 <= pw: the uniform 512 x 512 frame does; the 200 x 96 frame, whose Cartesian image is twice
    as wide as its beams are many, takes the dense kernel."""
    speckle = synth.make_frames(range(40, 46))
    det = ops.cfar(torch.from_numpy(speckle).cuda(), "SOCA", 20, 5, TAU_SOCA, gate=65)["mask"].cpu().numpy()
    rng = np.random.default_rng(1)
    for geo, masks, scatter in ((_geo("uniform"), det, True),
                                (_odd_geo(), (rng.random((5, 200, 96)) < 0.1).astype(np.uint8), False)):
        F, R, B = masks.shape
        pw, cw = R * ((B + 31) // 32), (geo.rows * geo.cols + 31) // 32  # polar / Cartesian bit-plane words
        assert ((cw + 1) // 2 <= pw) == scatter, (pw, cw)
        maps = _maps(gpu_ctx, geo, R, B)
        wants = [featx_ref.cart_points(m, geo) for m in masks]
        assert min(len(w[0]) for w in wants) > 100
        cap = max(len(w[0]) for w in wants)
        for kw in (dict(mask=torch.from_numpy(masks).cuda()), dict(bits=_bits(masks))):
            out = ops.cart_points(maps, capacity=cap, **kw)
            for f, (locs, pts) in enumerate(wants):
                k = int(out["count"][f])
                assert k == len(locs), (scatter, list(kw), f)
                assert np.array_equal(out["ij"][f, :k].cpu().numpy(), locs), (scatter, list(kw), f)
                assert np.array_equal(out["xy"][f, :k].cpu().numpy(), pts.astype(np.float32)), (scatter, list(kw), f)


def test_cart_points_odd_geometry(gpu_ctx):
    geo = _odd_geo()
    maps = _maps(gpu_ctx, geo, 200, 96)
    rng = np.random.default_rng(1)
    masks = (rng.random((5, 200, 96)) < 0.1).astype(np.uint8)
    out = ops.cart_points(maps, mask=torch.from_numpy(masks).cuda(), capacity=geo.rows * geo.cols)
    for f in range(5):
        locs, pts = featx_ref.cart_points(masks[f], geo)
        k = int(out["count"][f])
        assert k == len(locs) and np.array_equal(out["ij"][f, :k].cpu().numpy(), locs)
    empty = ops.cart_points(maps, mask=torch.zeros((2, 200, 96), dtype=torch.uint8, device="cuda"), capacity=8)
    assert empty["count"].tolist() == [0, 0]


# ------------------------------------------------------------------ cloud filters
def _pack(clouds):
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    pts = np.concatenate(clouds).astype(np.float32) if len(clouds) else np.zeros((0, 2), np.float32)
    return torch.from_numpy(pts).cuda(), torch.from_numpy(off).cuda(), off


def _clouds(rng, n_clouds, dim=2):
    out = []
    for c in range(n_clouds):
        n = int(rng.integers(0, 3000)) if c % 5 else int(rng.integers(0, 4))
        walls = synth.make_walls(rng, n_segments=6, extent=40.0)
        p = synth.sample_walls(rng, walls, n, 0.05) if n else np.zeros((0, 2))
        if n > 10:
            p[: n // 5] = rng.uniform(0, 40, (n // 5, 2))
        if dim == 3:
            p = np.c_[p, rng.normal(0, 0.3, n)]
        out.append(p.astype(np.float32))
    return out


def test_downsample_equals_oracle(gpu_ctx):
    rng = np.random.default_rng(3)
    clouds = _clouds(rng, 24) + [np.repeat(np.float32([[1.5, 2.5]]), 9, 0), np.float32([[0, 0], [0.3, 0.1]])]
    pts, off, off_h = _pack(clouds)
    for res in (0.5, 0.13, 7.0):
        out = ops.downsample(pts, off, max(len(c) for c in clouds), res)
        cnt = out["count"].cpu().numpy()
        for c, cl in enumerate(clouds):
            want, widx = orc.downsample(cl, res)
            assert cnt[c] == len(want), (c, res)
            s = off_h[c]
            assert np.array_equal(out["idx"][s:s + cnt[c]].cpu().numpy(), widx)
            assert np.array_equal(out["pts"][s:s + cnt[c]].cpu().numpy(), want)


def test_remove_outlier_equals_oracle(gpu_ctx):
    rng = np.random.default_rng(4)
    for dim in (2, 3):
        clouds = _clouds(rng, 16, dim)
        pts, off, off_h = _pack(clouds)
        for radius, mp in ((1.0, 5), (0.3, 1), (2.5, 40)):
            out = ops.remove_outlier(pts, off, max(len(c) for c in clouds), radius, mp)
            cnt = out["count"].cpu().numpy()
            for c, cl in enumerate(clouds):
                want, keep = orc.remove_outlier(cl, radius, mp) if len(cl) else (cl, np.zeros(0, bool))
                s = off_h[c]
                assert cnt[c] == len(want), (c, dim, radius)
                assert np.array_equal(out["pts"][s:s + cnt[c]].cpu().numpy(), want)
                assert np.array_equal(out["idx"][s:s + cnt[c]].cpu().numpy(), np.nonzero(keep)[0])


def test_match_equals_oracle(gpu_ctx):
    rng = np.random.default_rng(5)
    refs, ins = [], []
    for n_ref, n_in, spread in [(20000, 2000, 60.0), (300, 500, 5.0), (1, 10, 1.0), (5000, 100, 0.01), (0, 5, 1.0)]:
        refs.append(rng.uniform(0, spread, (n_ref, 2)).astype(np.float32))
        ins.append(rng.uniform(-0.2 * spread, 1.2 * spread, (n_in, 2)).astype(np.float32))
    refs.append(np.float32([[1, 0], [0, 1], [-1, 0], [1, 0]]))   # ties -> lowest index
    ins.append(np.float32([[0, 0], [1, 0]]))
    rp, ro, _ = _pack(refs)
    ip, io, io_h = _pack(ins)
    for md in (0.5, 10.0):
        out = ops.match(rp, ro, ip, io, max(len(r) for r in refs), md)
        for c in range(len(refs)):
            wi, wd = orc.match(refs[c], ins[c], md)
            s, e = io_h[c], io_h[c + 1]
            assert np.array_equal(out["ids"][s:e].cpu().numpy(), wi[0]), (c, md)
            assert np.array_equal(out["dists"][s:e].cpu().numpy(), wd[0])


# ------------------------------------------------------------------ ICP
def _pose(T):
    return np.array([T[0, 2], T[1, 2], np.arctan2(T[1, 0], T[0, 0])], np.float64)


def _run_icp_batch(pairs, guesses, prm):
    sp, so, _ = _pack([p[0] for p in pairs])
    tp, to, _ = _pack([p[1] for p in pairs])
    g = torch.from_numpy(np.stack(guesses).astype(np.float32)).cuda()
    out = ops.icp(sp, so, tp, to, g, max(len(p[0]) for p in pairs), max(len(p[1]) for p in pairs), prm)
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("mode", ["fixed20", "checkers"])
def test_icp_config3_pairs_match_oracle(gpu_ctx, mode):
    """BASELINE config 3: 2k-point source vs 20k-point target.  Tolerances are the north star's:
    1e-3 m / 1e-3 rad on the SE(2) pose, identical inlier count (and iteration count)."""
    kw = dict(smooth_length=0, max_iterations=20) if mode == "fixed20" else {}
    seeds = list(range(12))
    pairs = [synth.make_icp_pair(s)[:2] for s in seeds]
    guesses = [np.eye(3)] * len(pairs)
    got = _run_icp_batch(pairs, guesses, _lib.IcpParams(**kw))
    worst = 0.0
    for i, (src, tgt) in enumerate(pairs):
        want = orc.icp(src, tgt, None, orc.IcpParams(**kw))
        assert got["status"][i] == want["status"] == 0
        assert got["iterations"][i] == want["iterations"], (seeds[i], mode)
        assert got["inliers"][i] == want["inliers"], (seeds[i], mode)
        d = np.abs(_pose(got["T"][i]) - _pose(want["T"]))
        assert d[:2].max() < 1e-3 and d[2] < 1e-3, (seeds[i], d)
        worst = max(worst, d.max())
    print("worst pose deviation vs oracle:", worst)


def test_icp_small_clouds_guesses_and_shared_target(gpu_ctx):
    rng = np.random.default_rng(8)
    src, tgt, Tgt = synth.make_icp_pair(21, n_source=400, n_target=1500)
    guesses = [synth.se2(*rng.uniform(-0.3, 0.3, 2), rng.uniform(-0.05, 0.05)) for _ in range(30)]
    sp, so, _ = _pack([src])
    tp, to, _ = _pack([tgt])
    zero = torch.zeros(30, dtype=torch.int32, device="cuda")
    out = ops.icp(sp, so, tp, to, torch.from_numpy(np.stack(guesses).astype(np.float32)).cuda(), len(src), len(tgt),
                  _lib.IcpParams(), src_id=zero, tgt_id=zero)
    for i, g in enumerate(guesses):
        want = orc.icp(src, tgt, g.astype(np.float32))
        assert int(out["status"][i]) == want["status"]
        assert int(out["iterations"][i]) == want["iterations"] and int(out["inliers"][i]) == want["inliers"]
        d = np.abs(_pose(out["T"][i].cpu().numpy()) - _pose(want["T"]))
        assert d[:2].max() < 1e-3 and d[2] < 1e-3


def test_icp_failures_keep_the_guess(gpu_ctx):
    src, tgt, _ = synth.make_icp_pair(5, n_source=200, n_target=500)
    far = synth.se2(100.0, 100.0, 0.3).astype(np.float32)
    bad = np.eye(3, dtype=np.float32)
    bad[0, 0] = 1.2
    pairs = [(src, tgt), (src, tgt), (src, tgt), (np.zeros((0, 2), np.float32), tgt), (src, np.zeros((0, 2), np.float32))]
    g = [far, far, bad, np.eye(3), np.eye(3)]
    a = _run_icp_batch(pairs[:1] + pairs[3:], [far, np.eye(3), np.eye(3)], _lib.IcpParams())
    assert a["status"].tolist() == [1, 1, 6] and np.array_equal(a["T"][0], far)
    b = _run_icp_batch(pairs[1:3], g[1:3], _lib.IcpParams(trim_ratio=-1.0))
    assert b["status"].tolist() == [2, 5] and np.array_equal(b["T"][0], far) and np.array_equal(b["T"][1], bad)
    lib = _lib.load()
    assert lib.sfe_icp_status_message(2) == b"ErrorMnimizer: no point to minimize"


def test_pcl_drop_in_module(gpu_ctx, tmp_path):
    """bruce_slam.pcl as slam.py / feature_extraction.py call it."""
    from sonar_slam_b200.bruce_slam import pcl
    rng = np.random.default_rng(9)
    pts = _clouds(rng, 2)[1].astype(np.float64)                     # float64 in, like the node's `points`
    out = pcl.downsample(pts, 0.5)
    want, widx = orc.downsample(pts, 0.5)
    assert out.dtype == np.float32 and np.array_equal(out, want)
    keys = np.arange(len(pts), dtype=np.float64)[:, None]
    o2, d2 = pcl.downsample(pts, keys, 0.5)
    assert np.array_equal(o2, want) and np.array_equal(d2[:, 0], widx.astype(np.float32))
    assert np.array_equal(pcl.remove_outlier(out, 1.0, 5), orc.remove_outlier(out, 1.0, 5)[0])
    assert pcl.downsample(np.zeros((0, 2)), 0.5).shape == (0, 2)
    src, tgt, _ = synth.make_icp_pair(3, n_source=500, n_target=3000)
    ids, d = pcl.match(tgt, src, 1, 0.5)
    wi, wd = orc.match(tgt, src, 0.5)
    assert ids.shape == (1, 500) and ids.dtype == np.int32 and np.array_equal(ids, wi) and np.array_equal(d, wd)
    icp = pcl.ICP()
    with pytest.raises(RuntimeError):
        icp.compute(src, tgt, np.eye(3))
    cfg = tmp_path / "icp.yaml"
    cfg.write_text("""readingDataPointsFilters:

referenceDataPointsFilters:

matcher:
  KDTreeMatcher:
    knn: 1
    epsilon: 0
    maxDist: 10.0

outlierFilters:
  - MaxDistOutlierFilter:
      maxDist: 3.0
  - TrimmedDistOutlierFilter:
      ratio: 0.8

errorMinimizer:
  PointToPointErrorMinimizer

transformationCheckers:
  - CounterTransformationChecker:
      maxIterationCount: 40
  - DifferentialTransformationChecker:
      minDiffRotErr: 0.01
      minDiffTransErr: 0.1
      smoothLength: 4

inspector:
  NullInspector
""")
    icp.loadFromYaml(str(cfg))
    msg, T = icp.compute(src, tgt, np.eye(3))
    want = orc.icp(src, tgt)
    assert msg == "success" == want["message"] and T.dtype == np.float32 and T.shape == (3, 3)
    assert np.abs(_pose(T) - _pose(want["T"])).max() < 1e-3
    msg, T = icp.compute(src, tgt, synth.se2(100, 100, 0))
    assert msg == "no outlier to filter" and np.allclose(T, synth.se2(100, 100, 0))
