"""GPU parity of the batched front end (one C-ABI call, host buffers) against the chained CPU oracle."""
import numpy as np
import pytest
import torch

from oracle import featx_ref, oracle as orc, pipeline_ref
from sonar_slam_b200 import _lib, pipeline, synth
from sonar_slam_b200.bruce_slam import conversions

pytestmark = pytest.mark.gpu


def _pose(T):
    return np.array([T[0, 2], T[1, 2], np.arctan2(T[1, 0], T[0, 0])], np.float64)


@pytest.mark.parametrize("mode", ["checkers", "fixed20", "plane"])
def test_frontend_host_call_equals_oracle_chain(gpu_ctx, mode):
    n = 14
    d = synth.make_trajectory_frames(n, seed=3)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(gpu_ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    kw = dict(smooth_length=0, max_iterations=20) if mode == "fixed20" else {}
    if mode == "plane":   # X1: point-to-plane minimiser (icp.yaml:18-19) inside the fused call
        kw = dict(minimizer=1, normals_knn=5)
    fe = pipeline.FrontEnd(gpu_ctx, maps, max_frames=32, icp=_lib.IcpParams(**kw), min_points=30)
    got = fe.run_host(frames, poses, chunk_frames=5)
    clouds, want = pipeline_ref.run(frames, poses, geo, min_points=30, icp_params=orc.IcpParams(**kw))
    # clouds (bit-exact): read them back from the device
    r = fe.results_dev()
    stride = r["cloud_stride"]
    xy = gpu_ctx.to_host(r["cloud_xy"], (n, stride, 2), np.float32)
    for i, c in enumerate(clouds):
        assert np.array_equal(xy[i, :len(c)], c), i
    assert np.array_equal(got["npoints"], [len(c) for c in clouds])
    n_matched = 0
    for i in range(n):
        assert got["status"][i] == want[i]["status"], (i, got["status"][i], want[i]["status"])
        if want[i]["status"] == 0:
            n_matched += 1
            assert got["iterations"][i] == want[i]["iterations"], i
            assert got["inliers"][i] == want[i]["inliers"], i
            # default ICP mode = the oracle's accumulation order: the whole chain is bit-identical
            assert np.array_equal(got["T"][i].view(np.uint32), want[i]["T"].view(np.uint32)), (i, got["T"][i], want[i]["T"])
        else:
            assert np.allclose(got["T"][i], want[i]["T"])      # failed / skipped: the guess comes back
    assert got["status"][0] == 7 and n_matched >= n - 4
    # device-resident flavour gives the same answers
    dev_frames = torch.from_numpy(frames).cuda()
    fe.run_dev(dev_frames.data_ptr(), poses, n)
    gpu_ctx.sync()
    again = fe.run_host(frames, poses, chunk_frames=64)
    for k in ("status", "iterations", "inliers", "npoints"):
        assert np.array_equal(again[k], got[k])
    assert np.array_equal(again["T"], got["T"])


def test_frontend_both_icp_size_classes(gpu_ctx):
    """The front end serves ICP with two launches by problem size (pipeline.cu: FE_ICP_SMALL_*).  A finer voxel
    grid gives clouds on both sides of the 640-point class boundary; every frame must still equal the oracle."""
    n = 10
    d = synth.make_trajectory_frames(n, seed=5)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(gpu_ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    prm = dict(smooth_length=0, max_iterations=20)
    fe = pipeline.FrontEnd(gpu_ctx, maps, max_frames=16, icp=_lib.IcpParams(**prm), min_points=30, resolution=0.35,
                           submap_resolution=0.35, cap_source=4096, cap_target=12288)
    got = fe.run_host(frames, poses, chunk_frames=4)
    clouds, want = pipeline_ref.run(frames, poses, geo, min_points=30, submap_resolution=0.35,
                                    icp_params=orc.IcpParams(**prm), resolution=0.35)
    sizes = np.array([len(c) for c in clouds])
    assert np.array_equal(got["npoints"], sizes)
    assert (sizes > 640).any() and (sizes <= 640).any(), sizes  # both launches had work
    for i in range(n):
        assert got["status"][i] == want[i]["status"], (i, got["status"][i], want[i]["status"])
        if want[i]["status"] == 0:
            assert got["iterations"][i] == want[i]["iterations"] and got["inliers"][i] == want[i]["inliers"], i
            assert np.array_equal(got["T"][i].view(np.uint32), want[i]["T"].view(np.uint32)), (i, got["T"][i], want[i]["T"])


def test_frontend_equals_node_chain_with_slam_sign_convention(gpu_ctx, icp_yaml):
    """The reference's two nodes, call by call: FeatureExtraction.callback (drop-in mirror, GPU kernels through the
    host C ABI) publishes [p0, 0, p1] (feature_extraction.py:182); the SLAM node reads (x, -z) = (p0, -p1)
    (slam_ros.py:169-170), keeps it as the keyframe cloud, builds the window submap with get_points and calls
    compute_icp with the odometry guess.  The fused batch call must return the same edge for every frame --
    i.e. it applies the same lateral sign flip (sfe_frontend_params.flip_lateral = 1)."""
    from sonar_slam_b200.bruce_slam.feature_extraction import FeatureExtraction
    from sonar_slam_b200.bruce_slam.slam import SLAM, Pose2
    n = 9
    d = synth.make_trajectory_frames(n, seed=8)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    fx = FeatureExtraction()
    fx.init_node({"CFAR": {"Ntc": 40, "Ngc": 10, "Pfa": 0.1, "rank": 10, "alg": "SOCA"},
                  "filter": {"threshold": 65, "resolution": 0.5, "radius": 1.0, "min_points": 5, "skip": 1},
                  "compressed_images": False})
    slam = SLAM()
    slam.icp.loadFromYaml(icp_yaml)                                        # slam_ros.py: the node loads icp.yaml

    class KF:
        def __init__(self, points, pose):
            self.points, self.pose = points, pose

    edges = []
    for i in range(n):
        ping = synth.Ping(ping_id=i, image=frames[i], range_resolution=30.0 / 512, num_ranges=512, bearings=d["bearings"])
        pts = fx.callback(ping)                                            # feature node
        # the hand-off as the nodes do it: PointCloud2 [p0, 0, p1] (feature_extraction.py:181-190, float32 on the
        # wire) read back as (x, -z) (slam_ros.py:169-170) -- bruce_slam/conversions.py, same bytes without ROS
        points = conversions.keyframe_points(fx.feature_msg)
        assert fx.feature_msg.width == len(pts) and fx.feature_msg.point_step == 12
        slam.keyframes.append(KF(points, Pose2(*poses[i])))
        if i == 0:
            edges.append(None)
            continue
        window = list(range(max(0, i - 3), i))
        target = slam.get_points(window, i - 1)                            # slam.py:632-633
        guess = slam.keyframes[i - 1].pose.between(slam.keyframes[i].pose)
        if len(points) < 30 or len(target) < 30:
            edges.append(None)
            continue
        edges.append(slam.compute_icp(points, target, guess))
    fe = pipeline.FrontEnd(gpu_ctx, fx.device_maps(gpu_ctx, 512), max_frames=16, min_points=30)
    got = fe.run_host(frames, poses, chunk_frames=4)
    r = fe.results_dev()
    xy = gpu_ctx.to_host(r["cloud_xy"], (n, r["cloud_stride"], 2), np.float32)
    n_edges = 0
    for i in range(n):
        kf = slam.keyframes[i].points
        assert np.array_equal(xy[i, :len(kf)], kf.astype(np.float32)), i   # the keyframe cloud, sign flip included
        if edges[i] is None:
            assert got["status"][i] == 7
            continue
        msg, pose = edges[i]
        assert (msg == "success") == (got["status"][i] == 0), (i, msg, got["status"][i])
        if msg == "success":
            n_edges += 1
            dlt = np.abs(_pose(got["T"][i]) - np.array([pose.x(), pose.y(), pose.theta()]))
            assert dlt[:2].max() < 1e-3 and dlt[2] < 1e-3, (i, dlt)
    assert n_edges >= n - 3
    # with the odometry in the same (standard) frame as the flipped clouds the edges stay close to the odometry;
    # without the flip the clouds are mirrored against it
    off = pipeline.FrontEnd(gpu_ctx, fx.device_maps(gpu_ctx, 512), max_frames=16, min_points=30, flip_lateral=0)
    raw = off.run_host(frames, poses, chunk_frames=4)
    ro = off.results_dev()
    xy0 = gpu_ctx.to_host(ro["cloud_xy"], (n, ro["cloud_stride"], 2), np.float32)
    k = int(got["npoints"][2])
    assert np.array_equal(xy0[2, :k] * np.array([1, -1], np.float32), xy[2, :k])
    assert np.array_equal(raw["npoints"], got["npoints"])


def test_oversize_frames_report_too_large_with_small_capacities(gpu_ctx):
    """cap_source / cap_target below the first ICP size class: there is no second launch, so the one launch must
    itself report clouds beyond the capacities (SFE_ICP_TOO_LARGE = 8) and hand the guess back."""
    n = 8
    d = synth.make_trajectory_frames(n, seed=3)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(gpu_ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    clouds, _ = pipeline_ref.run(frames, poses, geo, min_points=30)
    sizes = np.array([len(c) for c in clouds])
    cap_s = int(np.sort(sizes)[n // 2])                          # about half of the frames exceed it
    fe = pipeline.FrontEnd(gpu_ctx, maps, max_frames=n, min_points=30, cap_source=cap_s, cap_target=1536)
    got = fe.run_host(frames, poses, chunk_frames=3)
    clouds, want = pipeline_ref.run(frames, poses, geo, min_points=30)
    assert (sizes > cap_s).any() and (sizes[1:] <= cap_s).any()
    for i in range(1, n):
        if sizes[i] > cap_s:
            assert got["status"][i] == 8 and got["iterations"][i] == 0 and got["inliers"][i] == 0, (i, got["status"][i])
            assert np.array_equal(got["T"][i], want[i]["T"] if want[i]["status"] != 0 else
                                  pipeline_ref.between(poses[i - 1], poses[i]))
        else:
            assert got["status"][i] == want[i]["status"], i
    fe2 = pipeline.FrontEnd(gpu_ctx, maps, max_frames=n, min_points=30, cap_source=640, cap_target=200)
    got2 = fe2.run_host(frames, poses, chunk_frames=8)
    assert (got2["status"][2:] == 8).all()                       # every window submap exceeds 200 points


def test_carried_window_stitches_batches(gpu_ctx):
    """Row N3 (submaps resident between calls): a replay fed in pieces with sfe_frontend_set_carry gives, frame for
    frame and bit for bit, the results of feeding it in one call -- the last `window` clouds and poses stay on the
    device and serve the first frames of the next call; without carry every piece starts cold."""
    n = 26
    d = synth.make_trajectory_frames(n, seed=12)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(gpu_ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    fe = pipeline.FrontEnd(gpu_ctx, maps, max_frames=32, min_points=30)
    whole = {k: v.copy() for k, v in fe.run_host(frames, poses, chunk_frames=7).items()}
    fe.set_carry(True)
    pieces = [(0, 9), (9, 10), (10, 12), (12, 26)]            # a one-frame and a two-frame piece: shorter than the window
    for j, (a, b) in enumerate(pieces):
        if j % 2 == 0:
            got = fe.run_host(frames[a:b], poses[a:b], chunk_frames=4)
        else:                                                  # device-resident flavour in between
            dev = torch.from_numpy(frames[a:b]).cuda()
            fe.run_dev(dev.data_ptr(), poses[a:b], b - a)
            r = fe.results_dev()
            got = dict(T=gpu_ctx.to_host(r["T"], (b - a, 3, 3), np.float32),
                       status=gpu_ctx.to_host(r["status"], (b - a,), np.int32),
                       iterations=gpu_ctx.to_host(r["iterations"], (b - a,), np.int32),
                       inliers=gpu_ctx.to_host(r["inliers"], (b - a,), np.int32))
        for k in ("status", "iterations", "inliers"):
            assert np.array_equal(got[k], whole[k][a:b]), (k, a, b)
        assert np.array_equal(got["T"].view(np.uint32), whole["T"][a:b].view(np.uint32)), (a, b)
    # carry off: the next piece starts cold again
    fe.set_carry(False)
    cold = fe.run_host(frames[12:26], poses[12:26], chunk_frames=8)
    assert cold["status"][0] == 7 and np.array_equal(cold["T"][3:], whole["T"][15:26])
    assert not np.array_equal(cold["T"][1], whole["T"][13])   # a two-frame window instead of three


def test_carried_run_dev_calls_back_to_back(gpu_ctx):
    """Three run_dev calls with the window carried across them, enqueued without a host sync in between: the next
    call's pose upload (double-buffered pinned staging) and feature stages must not overtake the previous call's scan
    match or carry copies.  The pieces shrink, so afterwards the result slots hold frames of all three calls -- slot i
    frame 230 + i, 140 + i or i -- each as one run_host call over the whole sequence computes it."""
    n, pieces = 270, [(0, 140), (140, 230), (230, 270)]
    d = synth.make_trajectory_frames(n, seed=4)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(gpu_ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    whole = pipeline.FrontEnd(gpu_ctx, maps, max_frames=n, min_points=30).run_host(frames, poses, clouds=True)
    fe = pipeline.FrontEnd(gpu_ctx, maps, max_frames=n, min_points=30)
    fe.set_carry(True)
    dev = torch.from_numpy(frames).cuda()
    for a, b in pieces:
        fe.run_dev(dev[a:].data_ptr(), poses[a:b], b - a)
    m = pieces[0][1]
    frame = np.concatenate([np.arange(230, 270), np.arange(180, 230), np.arange(90, 140)])
    r = fe.results_dev()
    assert np.array_equal(gpu_ctx.to_host(r["T"], (m, 9), np.float32).view(np.uint32),
                          whole["T"].reshape(n, 9)[frame].view(np.uint32))
    for k in ("iterations", "inliers", "status"):
        assert np.array_equal(gpu_ctx.to_host(r[k], (m,), np.int32), whole[k][frame]), k
    assert np.array_equal(gpu_ctx.to_host(r["cloud_count"], (m,), np.int32), whole["npoints"][frame])
    xy = gpu_ctx.to_host(r["cloud_xy"], (m, r["cloud_stride"], 2), np.float32).view(np.uint32)
    off = whole["cloud_offsets"]
    for i, f in enumerate(frame):
        assert np.array_equal(xy[i, :off[f + 1] - off[f]], whole["clouds"][off[f]:off[f + 1]].view(np.uint32)), i
    assert whole["status"][230] != 7 and (whole["status"] == 0).sum() >= n // 2   # a carried window; matches
