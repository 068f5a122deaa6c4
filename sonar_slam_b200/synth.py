"""Seeded synthetic inputs for the sonar front end (SURVEY.md section 8(d)).

The reference ships no data (its README points at a rosbag on Google Drive), so
every test / bench input is generated here:

  make_frame(seed)        one uint8 polar sonar image [num_ranges, num_beams]:
                          Rayleigh speckle plus a few bright range-arcs
  bearings_uniform / bearings_oculus
                          int16 centi-degree beam tables (the OculusPing.bearings
                          field read at feature_extraction.py:146,157)
  Ping                    ROS-free stand-in for the OculusPing fields the hot path
                          reads (feature_extraction.py:142-146,201,217)
  make_walls / make_icp_pair
                          2-D wall scene, (source, target, ground truth) scan pairs
  make_map_cloud          whole-map cloud: walls re-observed from keyframes along a trajectory
  make_trajectory_frames  frames seen from a moving vehicle (pipeline replay)
"""
from dataclasses import dataclass

import numpy as np


@dataclass
class Ping:
    """Fields of sonar_oculus/OculusPing that the feature extractor reads."""
    ping_id: int
    image: np.ndarray            # uint8 [num_ranges, num_beams], row 0 = nearest range
    range_resolution: float      # metres per range bin
    num_ranges: int
    bearings: np.ndarray         # int16 centi-degrees, ascending, one per beam
    stamp: float = 0.0


def bearings_uniform(num_beams=512, half_aperture_cdeg=6500):
    return np.round(np.linspace(-half_aperture_cdeg, half_aperture_cdeg, num_beams)).astype(np.int16)


def bearings_oculus(num_beams=512, half_aperture_deg=65.0):
    """Non-uniform table: beams equally spaced in sin(bearing), like the real head."""
    s = np.sin(np.deg2rad(half_aperture_deg))
    b = np.rad2deg(np.arcsin(np.linspace(-s, s, num_beams))) * 100.0
    return np.round(b).astype(np.int16)


def make_frame(seed, num_ranges=512, num_beams=512, n_arcs=6, sigma=18.0):
    """Config-1 style frame: clip(rayleigh(sigma)) + `n_arcs` arcs, 3 bins thick."""
    rng = np.random.default_rng(seed)
    img = rng.rayleigh(sigma, size=(num_ranges, num_beams))
    for _ in range(n_arcs):
        r0 = int(rng.integers(30, num_ranges - 33))
        w = int(rng.integers(30, 111))
        b0 = int(rng.integers(0, max(1, num_beams - w)))
        amp = rng.uniform(90.0, 200.0)
        img[r0:r0 + 3, b0:b0 + w] += amp
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def make_frames(seeds, **kw):
    return np.stack([make_frame(int(s), **kw) for s in seeds])


# ------------------------------------------------------------------ 2-D scenes / ICP pairs
def make_walls(rng, n_segments=120, extent=60.0, min_len=8.0, max_len=40.0):
    """Random wall segments (x0, y0, x1, y1) inside [0, extent]^2."""
    p0 = rng.uniform(0.0, extent, size=(n_segments, 2))
    ang = rng.uniform(0.0, 2 * np.pi, size=n_segments)
    ln = rng.uniform(min_len, max_len, size=n_segments)
    p1 = np.clip(p0 + np.c_[np.cos(ang), np.sin(ang)] * ln[:, None], 0.0, extent)
    return np.c_[p0, p1]


def sample_walls(rng, walls, n, sigma):
    seg_len = np.hypot(walls[:, 2] - walls[:, 0], walls[:, 3] - walls[:, 1])
    which = rng.choice(len(walls), size=n, p=seg_len / seg_len.sum())
    t = rng.uniform(0.0, 1.0, size=n)
    pts = walls[which, :2] + (walls[which, 2:] - walls[which, :2]) * t[:, None]
    return pts + rng.normal(0.0, sigma, size=pts.shape)


def make_map_cloud(n_points, seed=0, points_per_keyframe=360, sensor_range=30.0, sigma=0.05):
    """Whole-map cloud, what SLAM.get_points concatenates: wall segments re-observed from keyframes along a vehicle
    trajectory, `points_per_keyframe` wall points within `sensor_range` of every keyframe.  The scene grows with the
    run (about one 8-40 m wall per 12 000 points, ~250 points per 0.5 m cell on the walls).
    Returns (points float32 [n_points, 2] in world coordinates, keyframe index int32 [n_points],
    keyframe poses float64 [n_keyframes, 3] as x, y, theta)."""
    rng = np.random.default_rng(seed)
    n_segments = max(8, n_points // 12000)
    extent = 18.0 * np.sqrt(n_segments)
    walls = make_walls(rng, n_segments=n_segments, extent=extent)
    n_kf = -(-n_points // points_per_keyframe)
    s = np.linspace(0.0, 2 * np.pi, n_kf, endpoint=False)  # a closed loop through the scene, ridden once
    poses = np.c_[extent * (0.5 + 0.3 * np.cos(s)), extent * (0.5 + 0.3 * np.sin(2 * s)), s]
    pts, kf = [], []
    for k in range(n_kf):
        got = np.zeros((0, 2))
        while len(got) < points_per_keyframe:
            c = sample_walls(rng, walls, 8 * points_per_keyframe, sigma)
            got = np.r_[got, c[np.hypot(c[:, 0] - poses[k, 0], c[:, 1] - poses[k, 1]) < sensor_range]]
        pts.append(got[:points_per_keyframe])
        kf.append(np.full(points_per_keyframe, k, np.int32))
    return np.concatenate(pts)[:n_points].astype(np.float32), np.concatenate(kf)[:n_points], poses


def grid_thin(points, cell):
    """Keep the first point of every `cell`-sized square (order preserving)."""
    keys = np.floor(points / cell).astype(np.int64)
    keys = keys[:, 0] * 1000003 + keys[:, 1]
    _, first = np.unique(keys, return_index=True)
    return points[np.sort(first)]


def se2(x, y, theta):
    c, s = np.cos(theta), np.sin(theta)
    return np.array([[c, -s, x], [s, c, y], [0.0, 0.0, 1.0]])


def se3(t, axis, angle):
    """4x4 rigid transform: rotation by `angle` about the unit vector along `axis` (Rodrigues), then translation t."""
    k = np.asarray(axis, np.float64)
    k = k / np.linalg.norm(k)
    K = np.array([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + np.sin(angle) * K + (1.0 - np.cos(angle)) * (K @ K)
    T[:3, 3] = t
    return T


def make_icp_pair3(seed, n_source=2000, n_target=20000, extent=60.0, outlier_frac=0.2, max_t=1.0, max_rot=0.1,
                   sensor_range=30.0, half_aperture_deg=65.0, height=4.0, max_tilt=0.3):
    """Config-3 pair in 3-D: make_icp_pair's scene with walls `height` metres tall over an undulating floor.  Returns
    (source[N_s,3] f32, target[N_t,3] f32, T_gt 4x4 f64).

    target: wall and floor samples (sigma 0.03 m in x, y and z; a quarter on the floor), thinned on a 0.15 m voxel
            grid, in a frame centred on the sensor pose;
    source: wall and floor samples inside the sonar wedge (sigma 0.05 m) with `outlier_frac` outliers uniform in the wedge and
            in height, expressed in a frame displaced by T_gt^-1, so that T_gt maps source onto target.  T_gt turns by
            up to `max_rot` rad about an axis tilted up to `max_tilt` rad from z, and moves up to `max_t` m per axis.
    """
    rng = np.random.default_rng(seed)
    n_seg = max(6, int(48 * n_target / 20000))
    walls = make_walls(rng, n_segments=n_seg, extent=extent, min_len=15.0, max_len=50.0)

    def sample(n, sigma):  # wall points, and a quarter on an undulating floor (it pins z and the tilt)
        nf = n // 4
        xy = sample_walls(rng, walls, n - nf, sigma)
        walls_z = rng.uniform(0.0, height, n - nf)
        fxy = rng.uniform(0.0, extent, (nf, 2))
        floor_z = 0.4 * np.sin(fxy[:, 0] / 7.0) * np.cos(fxy[:, 1] / 5.0)
        return np.r_[np.c_[xy, walls_z], np.c_[fxy, floor_z]] + rng.normal(0.0, sigma, (n, 3))

    tgt = sample(4 * n_target, 0.03)
    keys = np.floor(tgt / 0.15).astype(np.int64)
    _, first = np.unique((keys[:, 0] * 1000003 + keys[:, 1]) * 1000003 + keys[:, 2], return_index=True)
    tgt = tgt[np.sort(first)]
    rng.shuffle(tgt)
    tgt = tgt[:n_target]
    pose = se2(rng.uniform(0.3, 0.5) * extent, rng.uniform(0.3, 0.7) * extent, rng.uniform(-0.5, 0.5))
    inv = np.linalg.inv(pose)
    to_sensor = lambda p: np.c_[p[:, :2] @ inv[:2, :2].T + inv[:2, 2], p[:, 2]]
    tgt_s = to_sensor(tgt)
    cand = to_sensor(sample(40 * n_source, 0.05))
    r = np.hypot(cand[:, 0], cand[:, 1])
    b = np.arctan2(cand[:, 1], cand[:, 0])
    cand = cand[(r < sensor_range) & (r > 0.5) & (np.abs(b) < np.deg2rad(half_aperture_deg))]
    n_in = int(round(n_source * (1.0 - outlier_frac)))
    if len(cand) < n_in:  # sparse view: pad with resampled structure points
        pad = cand[rng.integers(0, len(cand), n_in - len(cand))] if len(cand) else rng.uniform(-5, 5, (n_in, 3))
        cand = np.concatenate([cand, pad + rng.normal(0, 0.05, pad.shape)])
    src = cand[:n_in]
    rr = rng.uniform(0.5, sensor_range, n_source - n_in)
    bb = rng.uniform(-1, 1, n_source - n_in) * np.deg2rad(half_aperture_deg)
    src = np.concatenate([src, np.c_[rr * np.cos(bb), rr * np.sin(bb), rng.uniform(0.0, height, n_source - n_in)]])
    rng.shuffle(src)
    tilt, az = rng.uniform(0.0, max_tilt), rng.uniform(0.0, 2 * np.pi)
    axis = [np.sin(tilt) * np.cos(az), np.sin(tilt) * np.sin(az), np.cos(tilt)]
    T_gt = se3(rng.uniform(-max_t, max_t, 3), axis, rng.uniform(-max_rot, max_rot))
    Ti = np.linalg.inv(T_gt)
    src = src @ Ti[:3, :3].T + Ti[:3, 3]
    return src.astype(np.float32), tgt_s.astype(np.float32), T_gt


def make_icp_pair(seed, n_source=2000, n_target=20000, extent=60.0, outlier_frac=0.2,
                  max_t=1.0, max_rot=0.1, sensor_range=30.0, half_aperture_deg=65.0):
    """Config-3 pair.  Returns (source[N_s,2] f32, target[N_t,2] f32, T_gt 3x3 f64).

    target: wall samples (sigma 0.03 m), thinned on a 0.1 m grid, in a frame centred on
            the sensor pose;
    source: wall samples inside the sonar wedge (sigma 0.05 m) with `outlier_frac`
            uniform outliers, expressed in a frame displaced by T_gt^-1, so that
            T_gt maps source onto target (what ICP should recover from identity).
    """
    rng = np.random.default_rng(seed)
    n_seg = max(6, int(48 * n_target / 20000))
    walls = make_walls(rng, n_segments=n_seg, extent=extent, min_len=15.0, max_len=50.0)
    tgt = grid_thin(sample_walls(rng, walls, 4 * n_target, 0.03), 0.1)
    rng.shuffle(tgt)
    tgt = tgt[:n_target]
    # sensor pose in the scene
    pose = se2(rng.uniform(0.3, 0.5) * extent, rng.uniform(0.3, 0.7) * extent, rng.uniform(-0.5, 0.5))
    inv = np.linalg.inv(pose)
    to_sensor = lambda p: p @ inv[:2, :2].T + inv[:2, 2]
    tgt_s = to_sensor(tgt)
    cand = to_sensor(sample_walls(rng, walls, 40 * n_source, 0.05))
    r = np.hypot(cand[:, 0], cand[:, 1])
    b = np.arctan2(cand[:, 1], cand[:, 0])
    cand = cand[(r < sensor_range) & (r > 0.5) & (np.abs(b) < np.deg2rad(half_aperture_deg))]
    n_in = int(round(n_source * (1.0 - outlier_frac)))
    if len(cand) < n_in:  # sparse view: pad with resampled structure points
        cand = np.concatenate([cand, cand[rng.integers(0, max(1, len(cand)), n_in - len(cand))]
                               + rng.normal(0, 0.05, (n_in - len(cand), 2))]) if len(cand) else \
            rng.uniform(-5, 5, size=(n_in, 2))
    src = cand[:n_in]
    rr = rng.uniform(0.5, sensor_range, n_source - n_in)
    bb = rng.uniform(-1, 1, n_source - n_in) * np.deg2rad(half_aperture_deg)
    src = np.concatenate([src, np.c_[rr * np.cos(bb), rr * np.sin(bb)]])
    rng.shuffle(src)
    T_gt = se2(rng.uniform(-max_t, max_t), rng.uniform(-max_t, max_t), rng.uniform(-max_rot, max_rot))
    Ti = np.linalg.inv(T_gt)
    src = src @ Ti[:2, :2].T + Ti[:2, 2]
    return src.astype(np.float32), tgt_s.astype(np.float32), T_gt


# ------------------------------------------------------------------ frames seen from a moving vehicle
def make_trajectory_frames(n_frames, seed=0, num_ranges=512, num_beams=512, max_range=30.0, bearings=None,
                           device="cpu", step=0.35, odom_sigma=(0.03, 0.03, 0.004), sigma=18.0):
    """Synthetic "bag replay": a wall scene insonified from a vehicle moving along a smooth path.

    Returns dict(frames uint8 [n, num_ranges, num_beams] (torch, on `device`),
                 poses_true float64 [n,3], poses_odom float64 [n,3] (x, y, theta; odometry = truth +
                 integrated noise), bearings int16 centi-deg).
    Rendering (torch, runs on CPU or CUDA): wall sample points are moved into the sensor frame,
    binned to (range bin, beam) and given an echo amplitude; Rayleigh speckle everywhere.
    """
    import torch

    rng = np.random.default_rng(seed)
    if bearings is None:
        bearings = bearings_oculus(num_beams)
    b_rad = np.deg2rad(bearings.astype(np.float64) / 100.0)
    walls = make_walls(rng, n_segments=24, extent=90.0, min_len=15.0, max_len=45.0)
    seg_len = np.hypot(walls[:, 2] - walls[:, 0], walls[:, 3] - walls[:, 1])
    pts, amp = [], []
    for w, L in zip(walls, seg_len):
        m = int(L / 0.04)
        t = (np.arange(m) + 0.5) / m
        pts.append(w[:2] + (w[2:] - w[:2]) * t[:, None])
        amp.append(np.full(m, rng.uniform(110.0, 200.0)))
    pts, amp = np.concatenate(pts), np.concatenate(amp)
    # smooth path inside the scene
    th = 0.4 + np.cumsum(rng.normal(0, 0.01, n_frames)) + 0.15 * np.sin(np.arange(n_frames) / 40.0)
    xy = np.c_[np.cumsum(step * np.cos(th)), np.cumsum(step * np.sin(th))]
    xy = 45.0 + (xy - xy.mean(0)) * min(1.0, 35.0 / max(1e-9, np.abs(xy - xy.mean(0)).max()))
    poses_true = np.c_[xy, th]
    # odometry: per-step noise in the body frame, integrated
    odom = np.zeros_like(poses_true)
    odom[0] = poses_true[0]
    for i in range(1, n_frames):
        a, b = poses_true[i - 1], poses_true[i]
        c, s = np.cos(a[2]), np.sin(a[2])
        d = np.array([c * (b[0] - a[0]) + s * (b[1] - a[1]), -s * (b[0] - a[0]) + c * (b[1] - a[1]), b[2] - a[2]])
        d += rng.normal(0, odom_sigma)
        c, s = np.cos(odom[i - 1, 2]), np.sin(odom[i - 1, 2])
        odom[i] = [odom[i - 1, 0] + c * d[0] - s * d[1], odom[i - 1, 1] + s * d[0] + c * d[1], odom[i - 1, 2] + d[2]]

    dev = torch.device(device)
    P = torch.from_numpy(pts).to(dev)
    A = torch.from_numpy(amp).to(dev, torch.float32)
    bt = torch.from_numpy(b_rad).to(dev)
    res = max_range / num_ranges
    gen = torch.Generator(device=dev).manual_seed(int(seed))
    frames = torch.empty((n_frames, num_ranges, num_beams), dtype=torch.uint8, device=dev)
    chunk = 32 if dev.type == "cuda" else 8
    for f0 in range(0, n_frames, chunk):
        n = min(chunk, n_frames - f0)
        pose = torch.from_numpy(poses_true[f0:f0 + n]).to(dev)
        c, s = torch.cos(pose[:, 2])[:, None], torch.sin(pose[:, 2])[:, None]
        dx, dy = P[None, :, 0] - pose[:, 0:1], P[None, :, 1] - pose[:, 1:2]
        xs, ys = c * dx + s * dy, -s * dx + c * dy
        r, b = torch.hypot(xs, ys), torch.atan2(ys, xs)
        rb = torch.floor(r / res).long()
        bb = torch.searchsorted(bt, b.contiguous()).clamp_(0, num_beams - 1)
        ok = (rb >= 1) & (rb < num_ranges - 2) & (b > bt[0]) & (b < bt[-1])
        u = torch.rand((n, num_ranges, num_beams), device=dev, generator=gen).clamp_min_(1e-7)
        img = sigma * torch.sqrt(-2.0 * torch.log(u))
        fi = torch.arange(n, device=dev)[:, None].expand_as(rb)
        for dr in (0, 1):  # echoes are two range bins thick
            flat = (fi * num_ranges + rb + dr) * num_beams + bb
            img.view(-1).scatter_reduce_(0, flat[ok], A[None, :].expand_as(rb)[ok] + sigma, "amax")
        frames[f0:f0 + n] = torch.clamp(torch.round(img), 0, 255).to(torch.uint8)
    return dict(frames=frames, poses_true=poses_true, poses_odom=odom, bearings=bearings)
