"""The overlapped schedule of sfe_frontend_run_dev (sfe_frontend_set_overlap: feature stages of one sub-batch next to
the scan matching of the previous one, on two streams) gives bit for bit what the serial schedule gives."""
import numpy as np
import pytest
import torch

from oracle import featx_ref
from sonar_slam_b200 import _lib, pipeline, synth

pytestmark = pytest.mark.gpu

F = 300


@pytest.fixture(scope="module")
def replay(gpu_ctx):
    d = synth.make_trajectory_frames(F, seed=4)
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(gpu_ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    return dict(frames=d["frames"].cuda(), poses=d["poses_odom"], maps=maps)


def _results(ctx, fe, n):
    """Everything run_dev leaves on the device for its first n frames (blocking reads on the context's stream)."""
    r = fe.results_dev()
    out = {"T": ctx.to_host(r["T"], (n, 9), np.float32).view(np.uint32)}
    for k in ("iterations", "inliers", "status", "cloud_count"):
        out[k] = ctx.to_host(r[k], (n,), np.int32)
    xy = ctx.to_host(r["cloud_xy"], (n, r["cloud_stride"], 2), np.float32).view(np.uint32)
    out["clouds"] = [xy[i, :c] for i, c in enumerate(out["cloud_count"])]
    return out


def _assert_same(a, b, what):
    for k in ("T", "iterations", "inliers", "status", "cloud_count"):
        assert np.array_equal(a[k], b[k]), (what, k)
    for i, (x, y) in enumerate(zip(a["clouds"], b["clouds"])):
        assert np.array_equal(x, y), (what, "cloud", i)


def _run(ctx, fe, replay, n, sub_batch, **kw):
    fe.set_overlap(sub_batch)
    fe.run_dev(replay["frames"].data_ptr(), replay["poses"][:n], n, **kw)
    return _results(ctx, fe, n)


# 1 and 7: many sub-batches, 7 does not divide F; 256: two sub-batches, the second partial; 4096: larger than F
@pytest.mark.parametrize("sub_batch", [1, 7, 256, 4096])
def test_overlap_equals_serial(gpu_ctx, replay, sub_batch):
    fe = pipeline.FrontEnd(gpu_ctx, replay["maps"], max_frames=F, min_points=30,
                           icp=_lib.IcpParams(smooth_length=0, max_iterations=20))
    serial = _run(gpu_ctx, fe, replay, F, 0)
    assert (serial["status"] == 0).sum() >= F // 2          # the replay exercises the scan matcher
    _assert_same(_run(gpu_ctx, fe, replay, F, sub_batch), serial, sub_batch)
    _assert_same(_run(gpu_ctx, fe, replay, 5, sub_batch), _run(gpu_ctx, fe, replay, 5, 0), ("short", sub_batch))


def test_overlap_point_to_plane(gpu_ctx, replay):
    fe = pipeline.FrontEnd(gpu_ctx, replay["maps"], max_frames=F, min_points=30,
                           icp=_lib.IcpParams(minimizer=1, normals_knn=5))
    serial = _run(gpu_ctx, fe, replay, F, 0)
    assert (serial["status"] == 0).sum() >= F // 2
    _assert_same(_run(gpu_ctx, fe, replay, F, 64), serial, "plane")


def test_overlap_carry_back_to_back(gpu_ctx, replay):
    """Three calls with the window carried across them, enqueued without a host sync in between: the next call's
    pose upload and feature stages must not overtake the previous call's scan matching or carry copy.  The pieces
    shrink, so after the third call the result buffers still hold frames of all three."""
    pieces = [(0, 140), (140, 230), (230, 270)]

    def three_calls(sub_batch):
        fe = pipeline.FrontEnd(gpu_ctx, replay["maps"], max_frames=F, min_points=30)
        fe.set_overlap(sub_batch)
        fe.set_carry(True)
        for a, b in pieces:
            fe.run_dev(replay["frames"][a:].data_ptr(), replay["poses"][a:b], b - a)
        return _results(gpu_ctx, fe, pieces[0][1])

    serial = three_calls(0)
    assert serial["status"][0] != 7                          # the third call's first frame has a carried window
    for s in (7, 32):
        _assert_same(three_calls(s), serial, ("carry", s))


def test_overlap_feature_images_to_device(gpu_ctx, replay):
    n = 40
    fe = pipeline.FrontEnd(gpu_ctx, replay["maps"], max_frames=F, min_points=30)
    shape = (n, replay["maps"].rows, replay["maps"].cols, 3)
    img_serial = torch.zeros(shape, dtype=torch.uint8, device="cuda")
    img_overlap = torch.ones(shape, dtype=torch.uint8, device="cuda")
    serial = _run(gpu_ctx, fe, replay, n, 0, images=img_serial)
    _assert_same(_run(gpu_ctx, fe, replay, n, 16, images=img_overlap), serial, "images")
    assert torch.equal(img_serial, img_overlap)
