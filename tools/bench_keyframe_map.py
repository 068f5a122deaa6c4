"""SLAM.get_points on a growing map, host path against the device-resident keyframe map (bruce_slam.slam.KeyframeList).

Keyframes come from synth.make_map_cloud (360 points each) at 200, 600 and 2 000 keyframes (72 k to 720 k points).
After every pose has moved a little (an ISAM2 update), the calls the SLAM node makes per keyframe are timed on both
paths: the SSM target (last 3 frames relative to the previous keyframe, slam.py:632-633), the NSSM source (5 frames
in descending order, :857-860), the NSSM target (all but the last 8 keyframes, with keys) in world coordinates (:873)
and relative to a target keyframe (:999), and publish_point_cloud's whole map with keys (slam_ros.py:317-348).
Reports per call: the end-to-end median of both paths, the device time of the resident assemble (CUDA events around
sfe_keyframe_map_assemble_dev on resident data), bytes copied over PCIe by each path, and whether the outputs are
equal.  Prints one JSON line, with the card's name and power limit read in the same run.

    python tools/bench_keyframe_map.py [--reps 9] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
POINTS_PER_KEYFRAME = 360


def keyframes(n_kf, seed=1):
    import types
    from sonar_slam_b200 import synth
    from sonar_slam_b200.bruce_slam.slam import Pose2
    world, kf, poses = synth.make_map_cloud(n_kf * POINTS_PER_KEYFRAME, seed=seed)
    out = []
    for k, (x, y, t) in enumerate(poses):
        c, s = np.cos(t), np.sin(t)
        local = ((world[kf == k] - [x, y]) @ np.array([[c, -s], [s, c]])).astype(np.float32)
        out.append(types.SimpleNamespace(points=local, pose=Pose2(x, y, t)))
    return out


def calls(n):
    """(name, frames, ref_frame, return_keys) of the node's per-keyframe get_points calls, newest keyframe n - 1."""
    return [("ssm_target", list(range(n - 4, n - 1)), n - 2, False),
            ("nssm_source", list(range(n - 1, n - 6, -1)), n - 1, False),
            ("nssm_target_world", list(range(n - 8)), None, True),
            ("nssm_target_relative", list(range(n - 8)), n // 2, True),
            ("publish_map", None, None, True)]


def bytes_host(n_in):
    """sfe_downsample_host (api.cu: cloud_filter_host): points and offsets in, count, all n points and indices out."""
    return 8 * n_in + 8 + 4 + 8 * n_in + 4 * n_in


def bytes_resident(k, m, keys):
    """sfe_keyframe_map_assemble_host: the entry table (9 words per entry, 3 more) in, count and the m kept rows out."""
    return 4 * (9 * k + 3) + 4 + 8 * m + (4 * m if keys else 0)


def device_ms(km, slots, keys, tf, n_in, reps):
    """Median of CUDA-event-timed sfe_keyframe_map_assemble_dev calls on a map bound to torch's current stream."""
    import torch
    dev = torch.device("cuda", 0)
    pts = torch.empty((n_in, 2), dtype=torch.float32, device=dev)
    kout = torch.empty((n_in,), dtype=torch.float32, device=dev) if keys is not None else None
    m = torch.empty((1,), dtype=torch.int32, device=dev)
    slots = np.ascontiguousarray(slots, np.int32)
    from sonar_slam_b200 import _lib
    kk = None if keys is None else np.ascontiguousarray(keys, np.float32)

    def once():
        _lib.check(km.lib.sfe_keyframe_map_assemble_dev(km.handle, _lib.ptr(slots), _lib.ptr(kk), _lib.ptr(tf),
                                                        len(slots), 0.5, n_in, ctypes.c_void_p(pts.data_ptr()),
                                                        None if kout is None else ctypes.c_void_p(kout.data_ptr()),
                                                        ctypes.c_void_p(m.data_ptr())), "assemble_dev")
    once()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        once()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def entries(slam, frames, ref_frame, keys):
    """The entry table get_points builds for the resident map (bruce_slam/slam.py: _get_points_resident)."""
    kfs = slam.keyframes
    frames = range(len(kfs)) if frames is None else frames
    ref = None if ref_frame is None else kfs[ref_frame].pose
    tf = np.empty((len(frames), 6), np.float32)
    for i, k in enumerate(frames):
        T = (ref.between(kfs[k].pose) if ref is not None else kfs[k].pose).matrix().astype(np.float32)
        tf[i] = T[0, 0], T[0, 1], T[1, 0], T[1, 1], T[0, 2], T[1, 2]
    slots = slam.keyframes.slots([kfs[k].points for k in frames])
    return slots, (np.asarray(frames, np.float64).astype(np.float32) if keys else None), tf


def run(n_kf, reps):
    import torch
    from sonar_slam_b200 import ops
    from sonar_slam_b200.bruce_slam.slam import SLAM, Pose2
    from sonar_slam_b200.keyframe_map import KeyframeMap
    kfs = keyframes(n_kf)
    host, res = SLAM(), SLAM()
    host.keyframes = list(kfs)
    res.keyframes.extend(kfs)
    timed = SLAM()   # same clouds in a map on torch's stream, for the event timing of the assemble alone
    timed.keyframes.extend(kfs)
    timed.keyframes.map = KeyframeMap(ops.context(0))
    todo = calls(n_kf)
    for _, frames, ref, keys in todo:   # warm-up; uploads every cloud once
        host.get_points(frames, ref, keys)
        res.get_points(frames, ref, keys)
    uploaded = res.keyframes.map.size
    rng = np.random.default_rng(0)
    for kf in kfs:   # an ISAM2 update: every pose moves a little
        kf.pose = kf.pose.compose(Pose2(*(rng.normal(0, 1, 3) * [0.05, 0.05, 0.002])))
    out = {}
    for name, frames, ref, keys in todo:
        sel = range(n_kf) if frames is None else frames
        n_in = int(sum(len(kfs[k].points) for k in sel))
        t_host, t_res = [], []
        for _ in range(reps):   # the two paths alternate
            t0 = time.perf_counter()
            want = host.get_points(frames, ref, keys)
            t_host.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            got = res.get_points(frames, ref, keys)
            t_res.append((time.perf_counter() - t0) * 1e3)
        equal = (all(np.array_equal(a, b) and a.dtype == b.dtype for a, b in zip(got, want)) if keys
                 else np.array_equal(got, want))
        m = len(got[0] if keys else got)
        slots, kk, tf = entries(timed, frames, ref, keys)
        out[name] = dict(entries=len(sel), points_in=n_in, points_out=m,
                         host_ms=round(float(np.median(t_host)), 3), resident_ms=round(float(np.median(t_res)), 3),
                         assemble_device_ms=round(device_ms(timed.keyframes.map, slots, kk, tf, n_in, reps), 4),
                         host_bytes=bytes_host(n_in), resident_bytes=bytes_resident(len(sel), m, keys), equal=equal)
    torch.cuda.synchronize()
    return dict(keyframes=n_kf, points=uploaded[1], upload_once=res.keyframes.map.size == uploaded, calls=out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--sizes", default="200,600,2000")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_keyframe_map: no CUDA device (times are only measured on the GPU)")
    torch.cuda.set_device(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    res = dict(gpu=q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown", resolution=0.5,
               points_per_keyframe=POINTS_PER_KEYFRAME, maps=[run(int(n), args.reps) for n in args.sizes.split(",")])
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
