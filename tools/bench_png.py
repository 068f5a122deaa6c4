"""PNG compressed-ping decode (row N4) timing: the device PNG decoder (csrc/png.cu) next to cv2 on one host thread and
on every usable host core, and the front end fed with PNG pings (FrontEnd.run_png_host) next to the same front end fed
with the raw frames (FrontEnd.run_host).  Prints one JSON line and writes nothing.
Run on an H100:  PYTHONPATH=. python tools/bench_png.py [--frames N] [--device D]

Workload: N (default 4096) 512 x 512 synth.make_frame pings (64 seeds, cycled) written by cv2.imencode('.png') (8-bit
gray, Sub filter on every row: what image_transport's compressed plugin writes for a mono8 ping); the front-end legs
use 1024 synth.make_trajectory_frames frames written the same way.

  decode_frames_per_s     N / device decode time per call: the three stages below summed, CUDA events
                          (sfe_png_set_timing), mean of 5 calls after a warm-up
  stage_ms_*              those stages per call: check (IDAT CRC-32 + gather), inflate, unfilter (+ gray, Adler-32)
  call_frames_per_s       N / sfe_png_decode_to_dev wall time (host chunk walk and the copy of the IDAT bytes
                          included; median of 5)
  batch1_ms_median        one stream per call, wall time, median of 200
  h2d_ratio               compressed bytes / raw uint8 frame bytes
  cv2_ms_per_frame        cv2.imdecode(IMREAD_COLOR) + BGR2GRAY, one host thread
  cv2_all_cores_frames_per_s   the same over N frames in a process pool of len(os.sched_getaffinity(0)) workers
  run_png_host_fps / run_host_fps   front end on the same frames, chunk 256, median of 3 after a warm-up
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _gpu_name_and_power():
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception:  # noqa: BLE001
        import torch
        return torch.cuda.get_device_name(), "unknown"


def _cv2_decode_many(streams):
    import cv2
    cv2.setNumThreads(1)
    for b in streams:
        cv2.cvtColor(cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2GRAY)
    return len(streams)


def run(N, device=0, reps=5):
    import cv2
    import torch
    from oracle import featx_ref
    from sonar_slam_b200 import _lib, jpeg, ops, pipeline, png, synth
    torch.cuda.set_device(device)
    res = {}
    seeds = synth.make_frames(range(64))
    enc = [cv2.imencode(".png", seeds[i])[1].tobytes() for i in range(64)]
    streams = [enc[i % 64] for i in range(N)]
    buf, off = jpeg.pack(streams)
    ctx = ops.context(device)
    out = torch.empty((N, 512, 512), dtype=torch.uint8, device=f"cuda:{device}")
    st = np.empty(N, np.int32)

    def call():
        _lib.check(ctx.lib.sfe_png_decode_to_dev(ctx.handle, _lib.ptr(buf), _lib.ptr(off), N, 512, 512,
                                                 ops._dp(out), _lib.ptr(st)), "decode")
    call()
    assert (st == 0).all()
    for i in (0, N // 2, N - 1):
        assert np.array_equal(out[i].cpu().numpy(), seeds[i % 64])
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        call()
        ts.append(time.perf_counter() - t)
    res["call_frames_per_s"] = round(N / float(np.median(ts)), 1)
    res["call_ms"] = round(1e3 * float(np.median(ts)), 3)
    png.set_timing(True, ctx=ctx)
    for _ in range(reps):
        call()
    t = png.get_timing(ctx=ctx)
    png.set_timing(False, ctx=ctx)
    total = 0.0
    for k, (ms, _) in t.items():
        res[f"stage_ms_{k}"] = round(ms / reps, 3)
        total += ms / reps
    res["decode_ms"] = round(total, 3)
    res["decode_frames_per_s"] = round(N / (total / 1e3), 1)
    one_b, one_o = jpeg.pack(streams[:1])
    one = torch.empty((1, 512, 512), dtype=torch.uint8, device=f"cuda:{device}")
    s1 = np.empty(1, np.int32)
    lat = []
    for _ in range(220):
        t = time.perf_counter()
        _lib.check(ctx.lib.sfe_png_decode_to_dev(ctx.handle, _lib.ptr(one_b), _lib.ptr(one_o), 1, 512, 512,
                                                 ops._dp(one), _lib.ptr(s1)), "decode1")
        lat.append(time.perf_counter() - t)
    res["batch1_ms_median"] = round(1e3 * float(np.median(lat[20:])), 3)
    res["h2d_bytes_compressed"] = int(off[-1])
    res["h2d_bytes_raw"] = int(N * 512 * 512)
    res["h2d_ratio"] = round(int(off[-1]) / (N * 512 * 512), 4)
    cv2.setNumThreads(1)
    t = time.perf_counter()
    _cv2_decode_many(streams[:200])
    res["cv2_ms_per_frame"] = round(1e3 * (time.perf_counter() - t) / 200, 3)
    import multiprocessing as mp
    cores = len(os.sched_getaffinity(0))
    parts = [streams[i::cores] for i in range(cores)]
    with mp.get_context("spawn").Pool(cores) as pool:
        pool.map(_cv2_decode_many, [p[:2] for p in parts])  # workers started and cv2 imported
        t = time.perf_counter()
        pool.map(_cv2_decode_many, parts)
        res["cv2_all_cores_frames_per_s"] = round(N / (time.perf_counter() - t), 1)
    res["host_cores"] = cores
    res["device_beats_cv2_all_cores"] = res["decode_frames_per_s"] > res["cv2_all_cores_frames_per_s"]

    # front end: PNG pings vs raw frames
    n = 1024
    d = synth.make_trajectory_frames(n, seed=2)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    fb, fo = jpeg.pack([cv2.imencode(".png", f)[1].tobytes() for f in frames])
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    fe = pipeline.FrontEnd(ctx, maps, max_frames=n)
    a = fe.run_host(frames, poses)
    b = fe.run_png_host((fb, fo), poses)
    res["frontend_equal"] = all(np.array_equal(a[k], b[k]) for k in a)
    for name, fn in (("run_host_fps", lambda: fe.run_host(frames, poses)),
                     ("run_png_host_fps", lambda: fe.run_png_host((fb, fo), poses))):
        fn()
        ts = []
        for _ in range(3):
            t = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t)
        res[name] = round(n / float(np.median(ts)), 1)
    res["gpu"], res["power_limit"] = _gpu_name_and_power()
    return res


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    print(json.dumps(run(a.frames, a.device)))
