"""GPU: the front end's split down-sample (cloud.cu, downsample_cta_kernel behind ops.downsample_frames) compared
exactly (indices, order, float32 points, counts) with the CPU oracle, on the bench bag's raw clouds, on the edge cases
of its frame and submap classes, and on capacity launches whose workspace is in global memory."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from sonar_slam_b200 import ops, synth

pytestmark = pytest.mark.gpu

FRAME = 6144  # pipeline.cu, FE_DS_FRAME
SUBMAP = 2048  # pipeline.cu, FE_SUBMAP_SPLIT
MAX_POINTS = 65535  # cloud.cu, DSF_MAX_POINTS: the largest layout of the one-CTA kernel


def _check(clouds, res, frame_points=FRAME, n_max=None, with_cnt=True):
    """Packed at a fixed stride of n_max rows (as the front end packs them), down-sampled in one call."""
    n_max = n_max or max(max(len(c) for c in clouds), 1)
    pts = np.zeros((len(clouds) * n_max, 2), np.float32)
    for i, c in enumerate(clouds):
        pts[i * n_max:i * n_max + len(c)] = c
    cnt = torch.tensor([len(c) for c in clouds], dtype=torch.int32, device="cuda")
    if with_cnt:
        off = torch.arange(len(clouds) + 1, dtype=torch.int32, device="cuda") * n_max
    else:  # counts from the offsets: pack densely
        pts = np.concatenate([np.asarray(c, np.float32).reshape(-1, 2) for c in clouds])
        off = torch.tensor(np.r_[0, np.cumsum([len(c) for c in clouds])], dtype=torch.int32, device="cuda")
    r = ops.downsample_frames(torch.from_numpy(pts).cuda(), off, n_max, res, frame_points,
                              cnt=cnt if with_cnt else None)
    torch.cuda.synchronize()
    got_pts, got_idx, got_cnt = r["pts"].cpu().numpy(), r["idx"].cpu().numpy(), r["count"].cpu().numpy()
    off_h = off.cpu().numpy()
    for i, c in enumerate(clouds):
        want, widx = orc.downsample(np.asarray(c, np.float32).reshape(-1, 2), res) if len(c) else (np.zeros((0, 2)), [])
        o, k = off_h[i], got_cnt[i]
        assert k == len(want), (i, len(c), k, len(want))
        assert np.array_equal(got_idx[o:o + k], np.asarray(widx, np.int32)), (i, len(c))
        assert np.array_equal(got_pts[o:o + k].view(np.uint32), np.asarray(want, np.float32).view(np.uint32)), i


@pytest.fixture(scope="module")
def bag_raw():
    """Raw Cartesian clouds (CFAR -> remap -> nonzero, before any filter) of the first frames of bench.py's bag."""
    from oracle import featx_ref, pipeline_ref
    d = synth.make_trajectory_frames(48, seed=0)
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    return [pipeline_ref.frame_cloud(f, geo, resolution=0, min_points=1) for f in d["frames"].numpy()]


def test_bench_bag_raw_clouds(bag_raw):
    assert 2000 < np.mean([len(c) for c in bag_raw]) < FRAME
    _check(bag_raw, 0.5, n_max=8192)
    _check(bag_raw[:7], 0.5, with_cnt=False)


def test_empty_and_one_point_clouds(bag_raw):
    one = np.array([[3.25, -1.5]], np.float32)
    same = np.repeat(one, 3, axis=0)
    _check([np.zeros((0, 2), np.float32), one, bag_raw[0], same, np.zeros((0, 2), np.float32)], 0.5, n_max=8192)


def test_one_leaf_of_70_members():
    rng = np.random.default_rng(5)
    leaf = rng.uniform(10.0, 10.45, (70, 2)).astype(np.float32)  # the whole cloud one leaf (D = 0)
    fan = rng.uniform(-30, 30, (3000, 2)).astype(np.float32)
    # a 70-member leaf inside a D = 7 tree: the fan's bounding square is [-30, 30]^2, its leaves 0.47 m wide
    dense = np.concatenate([fan[:1500], rng.uniform(1.0, 1.4, (70, 2)).astype(np.float32), fan[1500:]])
    _check([leaf, dense, leaf[::-1].copy()], 0.5, n_max=8192)


@pytest.mark.parametrize("res", [4.0, 0.5, 0.1, 0.02])  # D = 4, 7, 10, 12 on a 60 m square (D > 7: wide keys)
def test_depths(bag_raw, res):
    _check(bag_raw[:6], res, n_max=8192)


def test_class_limit_and_capacity_launch():
    rng = np.random.default_rng(6)
    frame = 1024
    at = rng.uniform(-30, 30, (frame, 2)).astype(np.float32)
    past = rng.uniform(-30, 30, (frame + 1, 2)).astype(np.float32)
    big = rng.uniform(-30, 30, (3000, 2)).astype(np.float32)
    _check([at], 0.5, frame_points=frame, n_max=4096)
    _check([past], 0.5, frame_points=frame, n_max=4096)
    # a batch that mixes the two launches, and the front end's class on clouds either side of it
    _check([at, past, big, at[:10], np.zeros((0, 2), np.float32), big[::-1].copy()], 0.5, frame_points=frame,
           n_max=4096)
    near = rng.uniform(-30, 30, (FRAME + 1, 2)).astype(np.float32)
    _check([near[:FRAME], near, near[:100]], 0.5, n_max=8192)
    # n_max below the class: one launch of the frame kernel laid out for n_max
    _check([past, at[:7]], 0.5, frame_points=FRAME, n_max=frame + 1)


@pytest.mark.parametrize("res", [4.0, 0.5, 0.1, 0.02])  # D = 4, 7, 10, 12
def test_submap_class(bag_raw, res):
    """The front end's window submaps: clouds of up to FE_SUBMAP_SPLIT points in a launch laid out for them, the
    capacity launch laid out for 3 frames of 8192 points (workspace in global memory)."""
    clouds = [c[:SUBMAP] for c in bag_raw[:5]] + [bag_raw[5][:700], np.zeros((0, 2), np.float32), bag_raw[6][:SUBMAP + 1]]
    _check(clouds, res, frame_points=SUBMAP, n_max=3 * 8192)


def test_capacity_launch_in_global_memory():
    """Layouts above the shared-memory limit (about 13.9 k points on an H100) keep their workspace in global memory:
    clouds either side of the split, one of MAX_POINTS points, and a 15-level tree (two blobs 0.75 * res * 2^15
    apart)."""
    rng = np.random.default_rng(8)
    res = 0.5
    a = rng.uniform(0, 20 * res, (MAX_POINTS // 2, 2))
    b = rng.uniform(0, 20 * res, (MAX_POINTS - MAX_POINTS // 2, 2)) + 0.75 * res * 2 ** 15
    deep = np.concatenate([a, b]).astype(np.float32)
    wide = rng.uniform(-300, 300, (40000, 2)).astype(np.float32)
    small = rng.uniform(-30, 30, (3000, 2)).astype(np.float32)
    clouds = [small, deep, wide[:FRAME], np.zeros((0, 2), np.float32), wide, small[:1]]
    _check(clouds, res, frame_points=FRAME, n_max=MAX_POINTS)
    # both launches in global memory: the split itself above the shared-memory limit
    _check([wide, wide[:20000], deep[:30000], small], res, frame_points=20000, n_max=MAX_POINTS)


def test_capacity_layout_above_the_limit_is_rejected():
    from sonar_slam_b200 import _lib
    pts = torch.zeros((MAX_POINTS + 1, 2), dtype=torch.float32, device="cuda")
    off = torch.tensor([0, MAX_POINTS + 1], dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.SonarFEError, match="not supported"):
        ops.downsample_frames(pts, off, MAX_POINTS + 1, 0.5, FRAME)
