"""Packed feature clouds from the batched front end (sfe_frontend_set_clouds), the front end without its scan match
(sfe_frontend_set_scan_match) and FeatureExtraction.callback_batch, against the CPU oracle chain and the per-ping
paths."""
import ctypes
import itertools
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

from oracle import featx_ref, jpeg_ref, pipeline_ref  # noqa: E402
from sonar_slam_b200 import _lib, pipeline, synth  # noqa: E402

N = 40
KEYS = ("T", "iterations", "inliers", "status", "npoints")


@pytest.fixture(scope="module")
def bag(gpu_ctx):
    d = synth.make_trajectory_frames(N, seed=2)
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(gpu_ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    frames = d["frames"].numpy()
    oracle = {f: [pipeline_ref.slam_cloud(pipeline_ref.frame_cloud(x, geo), f) for x in frames] for f in (0, 1)}
    return types.SimpleNamespace(frames=frames, poses=d["poses_odom"], maps=maps, oracle=oracle,
                                 make=lambda **kw: pipeline.FrontEnd(gpu_ctx, maps, max_frames=N,
                                                                     **{"min_points": 30, **kw}))


def _frames_of(res):
    off = res["cloud_offsets"]
    return [res["clouds"][off[i]:off[i + 1]] for i in range(len(off) - 1)]


def _same_bytes(a, b):
    return len(a) == len(b) and np.ascontiguousarray(a, np.float32).tobytes() == \
        np.ascontiguousarray(b, np.float32).tobytes()


@pytest.mark.parametrize("flip", [0, 1])
@pytest.mark.parametrize("chunk", [1, 7, 256])
def test_run_host_clouds_equal_the_oracle(bag, flip, chunk):
    fe = bag.make(flip_lateral=flip)
    plain = fe.run_host(bag.frames, bag.poses, chunk_frames=chunk)
    res = fe.run_host(bag.frames, bag.poses, chunk_frames=chunk, clouds=True)
    for k in KEYS:
        assert np.array_equal(plain[k], res[k]), k
    assert res["cloud_offsets"][0] == 0 and np.array_equal(np.diff(res["cloud_offsets"]), res["npoints"])
    assert res["clouds"].dtype == np.float32 and res["clouds"].shape == (res["cloud_offsets"][-1], 2)
    for i, (got, want) in enumerate(zip(_frames_of(res), bag.oracle[flip])):
        assert _same_bytes(got, want), (flip, chunk, i)
    assert (res["status"] == 0).sum() > 10


def test_carry_in_pieces_gives_the_clouds_of_one_call(bag):
    one = bag.make()
    one.set_carry(True)
    whole = one.run_host(bag.frames, bag.poses, chunk_frames=7, clouds=True)
    fe = bag.make()
    fe.set_carry(True)
    parts = [fe.run_host(bag.frames[s], bag.poses[s], chunk_frames=7, clouds=True)
             for s in (slice(0, 13), slice(13, 14), slice(14, N))]
    assert _same_bytes(np.concatenate([p["clouds"] for p in parts]), whole["clouds"])
    for k in KEYS:
        assert np.array_equal(np.concatenate([p[k] for p in parts]), whole[k]), k


def test_geometry_jpeg_png_and_dev_flavours_give_the_run_host_clouds(bag, gpu_ctx):
    import torch
    jpg = [jpeg_ref.encode(f, q) for f, q in zip(bag.frames, itertools.cycle((80, 95)))]
    png = [cv2.imencode(".png", f)[1].tobytes() for f in bag.frames]
    decoded = np.stack([jpeg_ref.cv2_gray(b) for b in jpg])
    fe = bag.make()
    for frames, run in ((bag.frames, lambda: fe.run_host(list(bag.frames), bag.poses, chunk_frames=7,
                                                         geometry=np.zeros(N, np.int32), clouds=True)),
                        (decoded, lambda: fe.run_jpeg_host(jpg, bag.poses, chunk_frames=7, clouds=True)),
                        (bag.frames, lambda: fe.run_png_host(png, bag.poses, chunk_frames=7, clouds=True))):
        got = run()
        want = fe.run_host(frames, bag.poses, chunk_frames=7, clouds=True)
        assert np.array_equal(got["cloud_offsets"], want["cloud_offsets"])
        assert _same_bytes(got["clouds"], want["clouds"])
        for k in KEYS:
            assert np.array_equal(got[k], want[k]), k
    # run_dev: into its own device buffers, into the caller's, and against results_dev's strided clouds
    want = fe.run_host(bag.frames, bag.poses, clouds=True)
    dev_frames = torch.from_numpy(bag.frames).cuda()
    pts, off = fe.run_dev(dev_frames.data_ptr(), bag.poses, N, clouds=True)
    assert np.array_equal(off.cpu().numpy(), want["cloud_offsets"]) and _same_bytes(pts.cpu().numpy(), want["clouds"])
    total = int(want["cloud_offsets"][-1])
    mine = (torch.full((total, 2), 7.0, device="cuda"), torch.zeros(N + 1, dtype=torch.int64, device="cuda"))
    pts2, off2 = fe.run_dev(dev_frames.data_ptr(), bag.poses, N, clouds=mine)
    assert pts2.data_ptr() == mine[0].data_ptr() and _same_bytes(mine[0].cpu().numpy(), want["clouds"])
    assert np.array_equal(mine[1].cpu().numpy(), want["cloud_offsets"])
    r = fe.results_dev()
    stride, cnt = r["cloud_stride"], np.zeros(N, np.int32)
    _lib.check(gpu_ctx.lib.sfe_copy_to_host(gpu_ctx.handle, _lib.ptr(cnt), ctypes.c_void_p(r["cloud_count"]),
                                            cnt.nbytes), "copy")
    strided = np.zeros((N, stride, 2), np.float32)
    _lib.check(gpu_ctx.lib.sfe_copy_to_host(gpu_ctx.handle, _lib.ptr(strided), ctypes.c_void_p(r["cloud_xy"]),
                                            strided.nbytes), "copy")
    assert np.array_equal(cnt, want["npoints"])
    assert _same_bytes(np.concatenate([strided[i, :cnt[i]] for i in range(N)]), want["clouds"])


@pytest.mark.parametrize("cap_points", [8192, 5000])
def test_scan_match_off_host_and_dev_flavours(bag, gpu_ctx, cap_points):
    import torch
    on = bag.make(cap_points=cap_points)
    want = on.run_host(bag.frames, bag.poses, chunk_frames=7, clouds=True)
    fe = bag.make(cap_points=cap_points)
    fe.set_scan_match(False)
    fe.set_timing(True)
    got = fe.run_host(bag.frames, bag.poses, chunk_frames=7, clouds=True)
    timing = fe.get_timing()
    assert timing["submap"][1] == 0 and timing["icp"][1] == 0 and timing["cfar"][1] > 0
    assert _same_bytes(got["clouds"], want["clouds"]) and np.array_equal(got["npoints"], want["npoints"])
    too_large = want["status"] == _lib.ICP_TOO_LARGE
    assert np.array_equal(got["status"], np.where(too_large, _lib.ICP_TOO_LARGE, _lib.ICP_SKIPPED))
    assert too_large.any() == (cap_points == 5000)
    assert (got["iterations"] == 0).all() and (got["inliers"] == 0).all()
    assert np.array_equal(got["T"], np.broadcast_to(np.eye(3, dtype=np.float32), (N, 3, 3)))
    # the dev flavour
    dev_frames = torch.from_numpy(bag.frames).cuda()
    pts, off = fe.run_dev(dev_frames.data_ptr(), bag.poses, N, clouds=True)
    assert _same_bytes(pts.cpu().numpy(), want["clouds"])
    # with carry on the window advances without the scan match: turning it back on continues the sequence
    ref = bag.make(cap_points=cap_points)
    ref.set_carry(True)
    full = ref.run_host(bag.frames, bag.poses, chunk_frames=7)
    fe = bag.make(cap_points=cap_points)
    fe.set_carry(True)
    fe.set_scan_match(False)
    fe.run_host(bag.frames[:20], bag.poses[:20], chunk_frames=7)
    fe.set_scan_match(True)
    rest = fe.run_host(bag.frames[20:], bag.poses[20:], chunk_frames=7)
    for k in KEYS:
        assert np.array_equal(rest[k], full[k][20:]), k


def test_capacity_one_point_short_fails_and_exact_capacity_succeeds(bag, gpu_ctx):
    lib = gpu_ctx.lib
    fe = bag.make()
    fe.set_carry(True)
    total = int(fe.run_host(bag.frames, bag.poses, clouds=True)["cloud_offsets"][-1])
    # the same sequence again, fed twice: once failing, then retried; the failed call leaves the carried window alone
    ref, fe = bag.make(), bag.make()
    ref.set_carry(True), fe.set_carry(True)
    ref_a = ref.run_host(bag.frames[:20], bag.poses[:20], clouds=True)
    ref_b = ref.run_host(bag.frames[20:], bag.poses[20:], clouds=True)
    fe.run_host(bag.frames[:20], bag.poses[:20])
    need = int(ref_b["cloud_offsets"][-1])
    o = fe.alloc_results(N - 20)
    for cap, rc_want in ((need - 1, _lib.ERR_CAPACITY), (need, 0)):
        pts = np.full((need + 1, 2), 7.0, np.float32)
        off = np.full(N - 20 + 1, -1, np.int64)
        _lib.check(lib.sfe_frontend_set_clouds(fe.handle, _lib.ptr(pts), cap, _lib.ptr(off), 1), "set_clouds")
        rc = lib.sfe_frontend_run_host(fe.handle, _lib.ptr(np.ascontiguousarray(bag.frames[20:])),
                                       _lib.ptr(np.ascontiguousarray(bag.poses[20:])), N - 20, 7, _lib.ptr(o["T"]),
                                       _lib.ptr(o["iterations"]), _lib.ptr(o["inliers"]), _lib.ptr(o["status"]),
                                       _lib.ptr(o["npoints"]))
        lib.sfe_frontend_set_clouds(fe.handle, None, 0, None, 0)
        assert rc == rc_want, (cap, rc)
        assert np.array_equal(off, ref_b["cloud_offsets"])  # filled on failure too
        assert (pts[cap:] == 7.0).all()                      # nothing past the capacity
        if rc != 0:
            assert f"need {need} points" in lib.sfe_last_error().decode()
    assert _same_bytes(pts[:need], ref_b["clouds"])
    for k in KEYS:
        assert np.array_equal(o[k], ref_b[k]), k
    # the Python side retries once with the total the error reports
    fe2 = bag.make()
    got = fe2.run_host(bag.frames, bag.poses, clouds=5)
    assert int(got["cloud_offsets"][-1]) == total and len(got["clouds"]) == total
    # a destination of the wrong kind is refused before any device work
    pts = np.zeros((10, 2), np.float32)
    off = np.zeros(N + 1, np.int64)
    _lib.check(lib.sfe_frontend_set_clouds(fe2.handle, _lib.ptr(pts), 10, _lib.ptr(off), 1), "set_clouds")
    rc = lib.sfe_frontend_run_dev(fe2.handle, ctypes.c_void_p(1), _lib.ptr(bag.poses), N)
    lib.sfe_frontend_set_clouds(fe2.handle, None, 0, None, 0)
    assert rc == -1 and "host memory" in lib.sfe_last_error().decode()
    assert ref_a["cloud_offsets"][-1] + need == total


def _pings(seed, n, compressed):
    """A seeded synth bag: two geometries (512 range bins at 30 m, 384 at 20 m), one switch and back; compressed
    pings cycle JPEG, PNG and a progressive JPEG (which the device decoders refuse)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        R, res = (384, 20.0 / 384) if n // 3 <= i < 2 * n // 3 else (512, 30.0 / 512)
        img = synth.make_frame(int(rng.integers(1 << 30)), num_ranges=R)
        if compressed:
            kind = i % 3
            if kind == 0:
                data = jpeg_ref.encode(img, 85)
            elif kind == 1:
                data = cv2.imencode(".png", img)[1].tobytes()
            else:
                data = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
            image = types.SimpleNamespace(data=data)
        else:
            image = img
        p = synth.Ping(ping_id=i, image=image, range_resolution=res, num_ranges=R,
                       bearings=synth.bearings_uniform(512))
        p.header = types.SimpleNamespace(stamp=1000.0 + 0.1 * i)
        out.append(p)
    return out


@pytest.mark.parametrize("skip", [1, 3])
@pytest.mark.parametrize("compressed", [False, True])
def test_callback_batch_equals_per_ping_callback(gpu_ctx, skip, compressed):
    from sonar_slam_b200.bruce_slam.feature_extraction import FeatureExtraction
    params = {"CFAR": {"Ntc": 40, "Ngc": 10, "Pfa": 0.1, "rank": 10, "alg": "SOCA"},
              "filter": {"threshold": 65, "resolution": 0.5, "radius": 1.0, "min_points": 5, "skip": skip},
              "compressed_images": compressed}
    pings = _pings(7 + skip, 24, compressed)
    one, batch = FeatureExtraction(), FeatureExtraction()
    one.init_node(params), batch.init_node(params)
    want = []
    for p in pings:
        one.callback(p)
        want.append(one.feature_msg)
    got = batch.callback_batch(pings, max_frames=5)
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.data == w.data and g.width == w.width and g.point_step == w.point_step, i
        assert [(f.name, f.offset, f.datatype, f.count) for f in g.fields] == \
            [(f.name, f.offset, f.datatype, f.count) for f in w.fields], i
        assert g.header.stamp == w.header.stamp and g.header.frame_id == w.header.frame_id, i
    assert sum(w.width > 1 for w in want) > len(pings) // (2 * skip)
    assert batch.feature_msg is got[-1] and np.array_equal(batch.points, one.points, equal_nan=True)
