"""CPU-only: the host layer of SLAM.get_points' device-resident path (bruce_slam.slam.KeyframeList), with a numpy
stand-in for the device map (sonar_slam_b200.keyframe_map.KeyframeMap) built only from what the host layer passes --
wrong slots, keys or transform rows would show up as different points or keys than the host path gives."""
import os
import types

import numpy as np
import pytest

from oracle import oracle as orc
from sonar_slam_b200 import _lib, keyframe_map
from sonar_slam_b200.bruce_slam import pcl, slam

GOLD = os.path.join(os.path.dirname(__file__), "golden", "slam_host.npz")


class _FakeKeyframeMap:
    """sfe_keyframe_map's contract (include/sonarfe.h) in numpy: clouds copied in at append, every entry moved by its
    float32 row {r00, r01, r10, r11, tx, ty} as `points.dot(R.T) + t`, concatenated, down-sampled by the oracle."""
    made = []

    def __init__(self, ctx=None, capacity=0):
        self.clouds, self.appends = [], []
        _FakeKeyframeMap.made.append(self)

    def append(self, points):
        self.appends.append(list(points))
        first = len(self.clouds)
        self.clouds += [np.array(p, np.float32) for p in points]
        return np.arange(first, len(self.clouds), dtype=np.int32)

    @property
    def size(self):
        return len(self.clouds), sum(len(c) for c in self.clouds)

    def assemble(self, slots, keys, transforms, resolution, with_keys, device=False):
        pts, kk = [np.zeros((0, 2), np.float32)], [np.zeros(0, np.float32)]
        for k, (s, t) in enumerate(zip(slots, np.asarray(transforms, np.float32))):
            R = np.array([[t[0], t[1]], [t[2], t[3]]], np.float32)
            pts.append(self.clouds[s].dot(R.T) + t[4:6])
            kk.append(np.full(len(self.clouds[s]), keys[k] if with_keys else 0, np.float32))
        out, idx = orc.downsample(np.ascontiguousarray(np.concatenate(pts), np.float32), resolution)
        return (out, np.concatenate(kk)[idx]) if with_keys else out


@pytest.fixture()
def fake_map(monkeypatch):
    _FakeKeyframeMap.made = []
    monkeypatch.setattr(keyframe_map, "KeyframeMap", _FakeKeyframeMap)
    monkeypatch.setattr(_lib, "default_context", lambda: None)

    def downsample(points, *rest):   # the host path's pcl.downsample, served by the same oracle
        out, idx = orc.downsample(np.asarray(points, np.float32), rest[-1])
        return out if len(rest) == 1 else (out, np.asarray(rest[0], np.float32)[idx])

    monkeypatch.setattr(pcl, "downsample", downsample)
    return _FakeKeyframeMap


def _slams(g=None, n=4, seed=0):
    """(resident, host): two SLAM objects over the same keyframes, one in SLAM()'s KeyframeList, one in a plain list."""
    rng = np.random.default_rng(seed)
    if g is not None:
        kfs = [types.SimpleNamespace(points=g[f"kf{k}_points"], pose=slam.Pose2(*g[f"kf{k}_pose"])) for k in range(4)]
    else:
        kfs = [types.SimpleNamespace(points=rng.uniform(-20, 20, (int(rng.integers(1, 300)), 2)).astype(np.float32),
                                     pose=slam.Pose2(*rng.uniform(-1, 1, 3) * [30, 30, 3])) for _ in range(n)]
    res = slam.SLAM()
    res.keyframes.extend(kfs)
    host = slam.SLAM()
    host.keyframes = list(kfs)
    return res, host


def _same(a, b):
    if isinstance(a, tuple):
        return all(_same(x, y) for x, y in zip(a, b)) and len(a) == len(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


def test_slam_starts_with_the_resident_list():
    s = slam.SLAM()
    assert isinstance(s.keyframes, slam.KeyframeList) and isinstance(s.keyframes, list) and s.keyframes == []


def test_resident_host_layer_reproduces_the_reference_fixture(fake_map):
    g = np.load(GOLD)
    res, host = _slams(g)
    assert _same(res.get_points(), g["points_all"])
    assert _same(res.get_points([0, 1, 2], 3), g["points_ref_idx"])
    assert _same(res.get_points([1, 3], slam.Pose2(1.0, 0.5, -0.2)), g["points_ref_pose"])
    pts, keys = res.get_points([0, 2, 3], 1, True)
    assert _same(pts, g["points_keys_pts"]) and _same(keys, g["points_keys_keys"].astype(np.float32))
    assert _same((pts, keys), host.get_points([0, 2, 3], 1, True))
    assert len(fake_map.made) == 1 and len(fake_map.made[0].clouds) == 4   # every cloud uploaded once


@pytest.mark.parametrize("frames", [[0, 1, 2, 3], [3, 2, 1, 0], [2, 2, 0, 2], [-1, 0, -4, 1], "generator"])
@pytest.mark.parametrize("ref", [None, 2, -1, "pose"])
@pytest.mark.parametrize("keys", [False, True])
def test_resident_equals_host_path(fake_map, frames, ref, keys):
    """Any iterable in any order, repeats, negative indices (slot of the wrapped index, key as given), ref_frame as
    None / int / Pose2, keys on and off."""
    res, host = _slams(seed=3)
    ref = slam.Pose2(2.0, -1.0, 0.3) if ref == "pose" else ref
    frames = [1, -2] if frames == "generator" else frames
    got = res.get_points((k for k in frames), ref, keys)
    assert _same(got, host.get_points(frames, ref, keys))
    if keys:
        assert set(np.unique(got[1])) <= {np.float32(k) for k in frames}
    m = fake_map.made[0]
    assert len(m.clouds) == len(set(k % 4 for k in frames))   # each selected array once, repeats and aliases included


def test_negative_index_uses_the_wrapped_slot_and_the_given_key(fake_map):
    res, host = _slams(seed=5)
    pts, keys = res.get_points([-1], None, True)
    assert np.array_equal(fake_map.made[0].clouds[0], res.keyframes[3].points)
    assert len(keys) and np.all(keys == -1.0) and keys.dtype == np.float32 and keys.shape == (len(pts), 1)
    assert _same((pts, keys), host.get_points([-1], None, True))


def test_upload_is_lazy_once_per_array_and_follows_replaced_arrays(fake_map):
    res, host = _slams(seed=7)
    assert fake_map.made == []                       # nothing before the first call
    res.get_points([0, 1], None)
    m = fake_map.made[0]
    assert [len(a) for a in m.appends] == [2]
    res.get_points(None, 0, True)                    # one append for the two arrays not stored yet
    assert [len(a) for a in m.appends] == [2, 2] and m.appends[1][0] is res.keyframes[2].points
    for kf in res.keyframes:                         # poses changed (an ISAM2 update): nothing is uploaded again
        kf.pose = kf.pose.compose(slam.Pose2(0.1, -0.05, 0.01))
    assert _same(res.get_points(None, 1, True), host.get_points(None, 1, True))
    assert len(m.appends) == 2
    new = res.keyframes[1].points[::2].copy()        # a replaced .points array gets a slot of its own
    res.keyframes[1].points = new
    assert _same(res.get_points(), host.get_points())
    assert len(m.appends) == 3 and len(m.appends[2]) == 1 and m.appends[2][0] is new and len(m.clouds) == 5
    res.keyframes.append(types.SimpleNamespace(points=np.ones((5, 2), np.float32), pose=slam.Pose2(1, 2, 3)))
    host.keyframes.append(res.keyframes[-1])
    assert _same(res.get_points(None, None, True), host.get_points(None, None, True))
    assert len(m.appends) == 4 and m.size == (6, sum(len(c) for c in m.clouds))


def test_path_choice(fake_map):
    res, host = _slams(seed=9)
    host.get_points(None, 0, True)                   # a plain list: host path, no device map
    assert fake_map.made == []
    res.keyframes[2].points = res.keyframes[2].points.astype(np.float64)
    assert _same(res.get_points(None, 0, True), host.get_points(None, 0, True))
    assert fake_map.made == []                       # one float64 cloud: the whole call on the host, like numpy
    assert _same(res.get_points([0, 1, 3], 0), host.get_points([0, 1, 3], 0))
    assert len(fake_map.made) == 1                   # the float32 clouds alone: device map
    res.keyframes[0].points = np.asfortranarray(res.keyframes[0].points)   # float32 [N, 2] in any layout: device map
    assert _same(res.get_points([0, 1], 0), host.get_points([0, 1], 0))
    assert len(fake_map.made[0].appends) == 2 and fake_map.made[0].appends[1][0] is res.keyframes[0].points
    res.keyframes[1].points = res.keyframes[1].points.astype(np.float16)   # other dtypes stay on the host
    assert _same(res.get_points([0, 1], 0), host.get_points([0, 1], 0))
    assert len(fake_map.made[0].appends) == 2


def test_empty_selections_have_the_host_shapes(fake_map):
    res, host = _slams(seed=11)
    res.keyframes[1].points = host.keyframes[1].points = np.zeros((0, 2), np.float32)
    for frames in ([], [1], [1, 1]):
        for keys in (False, True):
            got, want = res.get_points(frames, 0, keys), host.get_points(frames, 0, keys)
            assert _same(got, want)
            if keys:
                assert got[0].shape == (0, 2) and got[1].shape == (0, 1) and got[1].dtype == np.float32
            else:
                assert got.shape == (0, 2) and got.dtype == np.float32
    assert fake_map.made == []                       # empty input comes straight back, as pcl.downsample's does
    assert _same(res.get_points([1, 0], None, True), host.get_points([1, 0], None, True))   # empty cloud among others


def test_out_of_range_index_raises_before_any_device_work(fake_map):
    res, host = _slams(seed=13)
    with pytest.raises(IndexError):
        host.get_points([0, 4])
    with pytest.raises(IndexError):
        res.get_points([0, 4])
    with pytest.raises(IndexError):
        res.get_points([0, -5], None, True)
    with pytest.raises(IndexError):
        res.get_points([0], 7)
    assert fake_map.made == []
