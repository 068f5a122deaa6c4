"""The front end's packed clouds and its feature-node mode, on bench.py's workload (the 4096-frame config-4 bag replay:
512 x 512 uint8 frames, CFAR SOCA 40/10 Pfa 0.1, gate 65, the 0.5 m voxel and outlier filters, window 3, ICP with 20
iterations).  Per step:
  run_dev        frames/s with the scan match on and off (CUDA events around K calls, frames resident on the device)
  run_host       frames/s without and with clouds (host clock around K calls, frames in pinned host memory)
  bytes_back     bytes copied back to the host per step, without and with clouds (computed from the results)
  callback       FeatureExtraction.callback per ping vs callback_batch on the bag's first 1024 pings (skip 1; host
                 clock, one warm-up pass each); the messages are checked byte for byte
Prints one JSON line with the card's name and power limit.

    python tools/bench_frontend_clouds.py [--steps K] [--warmup W] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
F, R, B, PINGS = 4096, 512, 512, 1024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_frontend_clouds.py: no CUDA device")
    from sonar_slam_b200 import _lib, ops, pipeline, synth
    from sonar_slam_b200.bruce_slam.feature_extraction import FeatureExtraction
    K, W = args.steps, args.warmup

    d = synth.make_trajectory_frames(F, seed=0, device="cuda:0")
    frames_dev, poses = d["frames"], d["poses_odom"]
    fx = FeatureExtraction()
    fx.generate_map_xy(synth.Ping(0, None, 30.0 / R, R, d["bearings"]))
    ctx = ops.context(0)
    maps = _lib.Maps(ctx, fx.map_x, fx.map_y, R, B, fx.width, fx.height)
    fe = pipeline.FrontEnd(ctx, maps, max_frames=F, icp=_lib.IcpParams(smooth_length=0, max_iterations=20))
    host_frames_t = torch.empty((F, R, B), dtype=torch.uint8, pin_memory=True)
    host_frames_t.copy_(frames_dev)
    host_frames = host_frames_t.numpy()

    def dev_fps(scan_match):
        fe.set_scan_match(scan_match)
        for _ in range(W):
            fe.run_dev(frames_dev.data_ptr(), poses, F)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(K):
            fe.run_dev(frames_dev.data_ptr(), poses, F)
        e1.record()
        torch.cuda.synchronize()
        fe.set_scan_match(True)
        return K * F / (e0.elapsed_time(e1) / 1e3)

    def host_fps(clouds):
        out = fe.alloc_results(F)
        for _ in range(W):
            res = fe.run_host(host_frames, poses, out=out, clouds=clouds)
        t0 = time.perf_counter()
        for _ in range(K):
            res = fe.run_host(host_frames, poses, out=out, clouds=clouds)
        return K * F / (time.perf_counter() - t0), res

    rows = {"run_dev_fps": {"scan_match_on": dev_fps(True), "scan_match_off": dev_fps(False)}}
    fps_plain, plain = host_fps(None)
    fps_clouds, packed = host_fps(True)
    for k in ("T", "iterations", "inliers", "status", "npoints"):
        assert np.array_equal(plain[k], packed[k]), k
    per_frame = sum(plain[k].nbytes for k in ("T", "iterations", "inliers", "status", "npoints"))
    rows["run_host_fps"] = {"without_clouds": fps_plain, "with_clouds": fps_clouds}
    rows["bytes_back_per_step"] = {"without_clouds": per_frame,
                                   "with_clouds": per_frame + packed["clouds"].nbytes + packed["cloud_offsets"].nbytes,
                                   "cloud_points": int(packed["cloud_offsets"][-1])}

    # the feature node on the bag's first pings: per-ping callback against callback_batch
    imgs = frames_dev[:PINGS].cpu().numpy()
    pings = [synth.Ping(i, imgs[i], 30.0 / R, R, d["bearings"]) for i in range(PINGS)]
    node = {"CFAR": {"Ntc": 40, "Ngc": 10, "Pfa": 0.1, "rank": 10, "alg": "SOCA"},
            "filter": {"threshold": 65, "resolution": 0.5, "radius": 1.0, "min_points": 5, "skip": 1}}
    one, batch = FeatureExtraction(), FeatureExtraction()
    one.init_node(node), batch.init_node(node)

    def per_ping():
        out = []
        for p in pings:
            one.callback(p)
            out.append(one.feature_msg)
        return out
    per_ping()
    t0 = time.perf_counter()
    want = per_ping()
    t_one = time.perf_counter() - t0
    batch.callback_batch(pings)
    t0 = time.perf_counter()
    got = batch.callback_batch(pings)
    t_batch = time.perf_counter() - t0
    assert all(g.data == w.data for g, w in zip(got, want)), "callback_batch differs from callback"
    rows["callback_pings_per_s"] = {"callback": PINGS / t_one, "callback_batch": PINGS / t_batch,
                                    "speedup": t_one / t_batch}

    p = torch.cuda.get_device_properties(0)
    try:
        pw = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                            capture_output=True, text=True).stdout.strip()
    except OSError:
        pw = None
    line = json.dumps(dict(gpu=p.name, power_limit_w=pw, frames=F, steps=K, **rows))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
