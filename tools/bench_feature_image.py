"""Feature-image timing (feature_extraction.py:226-228 on the device): the kernel (csrc/featx.cu: feature_image_kernel),
the host call, cv2 on one host thread and on every usable host core, and the front end with and without host-side
images.  Prints one JSON line and writes nothing.
Run on an H100:  PYTHONPATH=. python tools/bench_feature_image.py [--frames N] [--device D]

Workload: N (default 4096) 512 x 512 synth.make_frame pings (64 seeds, cycled) remapped into the 512 x 929 Cartesian
image of the Oculus bearing table, COLORMAP_JET; the front-end legs use 1024 synth.make_trajectory_frames frames.

  kernel_ms, kernel_frames_per_s   sfe_feature_image_dev on all N device frames, CUDA events, mean of 10 calls after
                                   a warm-up
  bytes_per_s, hbm_fraction        algorithmic bytes (N frames + the 8 B/pixel table once + N images) / kernel time,
                                   and that over the 3.35 TB/s data-sheet HBM3 bandwidth
  batch1_ms_median                 sfe_feature_image_host on one frame (copy in, kernel, copy out), median of 200
  cv2_ms_per_frame                 cv2.remap + applyColorMap(JET), one host thread
  cv2_all_cores_frames_per_s       the same over N frames in a process pool of len(os.sched_getaffinity(0)) workers
  run_host_fps, run_host_images_fps   FrontEnd.run_host, chunk 256, without / with images into a pinned host array,
                                      median of 3 after a warm-up
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12


def _gpu_name_and_power():
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in q.split(",")]
    return name, power


def _geometry():
    from oracle import featx_ref
    from sonar_slam_b200 import synth
    return featx_ref.Geometry(30.0 / 512, 512, synth.bearings_oculus(512))


def _cv2_many(frames):
    import cv2
    cv2.setNumThreads(1)
    geo = _geometry()
    for f in frames:
        cv2.applyColorMap(cv2.remap(f, geo.map_x, geo.map_y, cv2.INTER_LINEAR), 2)
    return len(frames)


def run(N, device=0, reps=10):
    import cv2
    import torch
    from oracle import featx_ref
    from sonar_slam_b200 import _lib, feature_image, ops, pipeline, synth
    torch.cuda.set_device(device)
    res = {}
    geo = _geometry()
    seeds = synth.make_frames(range(64))
    frames = np.stack([seeds[i % 64] for i in range(N)])
    ctx = ops.context(device)
    maps = _lib.Maps(ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    dev = torch.from_numpy(frames).cuda()
    ops.feature_image(dev, maps, ctx=ctx)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = ops.feature_image(dev, maps, ctx=ctx)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    npix = geo.rows * geo.cols
    nbytes = N * 512 * 512 + 8 * npix + N * npix * 3
    res.update(kernel_ms=ms, kernel_frames_per_s=N / ms * 1e3, bytes_per_s=nbytes / ms * 1e3,
               hbm_fraction=nbytes / ms * 1e3 / HBM_BYTES_PER_S, algorithmic_bytes=nbytes)
    k = [0, N // 2, N - 1]
    want = [cv2.applyColorMap(cv2.remap(frames[i], geo.map_x, geo.map_y, cv2.INTER_LINEAR), 2) for i in k]
    res["device_equals_cv2"] = bool(all(np.array_equal(out[i].cpu().numpy(), w) for i, w in zip(k, want)))
    del out

    one = np.ascontiguousarray(frames[:1])
    img = np.empty((1, geo.rows, geo.cols, 3), np.uint8)
    for _ in range(10):
        feature_image.render_host(maps, one, ctx=ctx, out=img)
    t = []
    for _ in range(200):
        t0 = time.perf_counter()
        feature_image.render_host(maps, one, ctx=ctx, out=img)
        t.append(time.perf_counter() - t0)
    res["batch1_ms_median"] = float(np.median(t) * 1e3)

    cv2.setNumThreads(1)
    _cv2_many(frames[:4])
    t0 = time.perf_counter()
    _cv2_many(frames[:64])
    res["cv2_ms_per_frame"] = (time.perf_counter() - t0) / 64 * 1e3
    import multiprocessing as mp
    workers = len(os.sched_getaffinity(0))
    parts = np.array_split(frames, workers)
    with mp.get_context("spawn").Pool(workers) as pool:
        pool.map(_cv2_many, [p[:2] for p in parts])
        t0 = time.perf_counter()
        pool.map(_cv2_many, parts)
        res["cv2_all_cores_frames_per_s"] = N / (time.perf_counter() - t0)
    res["host_cores"] = workers

    d = synth.make_trajectory_frames(1024, seed=2)
    tf, poses = d["frames"].numpy(), d["poses_odom"]
    tgeo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    tmaps = _lib.Maps(ctx, tgeo.map_x, tgeo.map_y, 512, 512, tgeo.width, tgeo.height)
    fe = pipeline.FrontEnd(ctx, tmaps, max_frames=len(tf))
    pinned = torch.empty((len(tf), tgeo.rows, tgeo.cols, 3), dtype=torch.uint8).pin_memory().numpy()
    for key, images in (("run_host_fps", None), ("run_host_images_fps", pinned)):
        fe.run_host(tf, poses, images=images)
        t = []
        for _ in range(3):
            t0 = time.perf_counter()
            r = fe.run_host(tf, poses, images=images)
            t.append(time.perf_counter() - t0)
        res[key] = len(tf) / float(np.median(t))
        res[key.replace("fps", "status_ok")] = int((r["status"] == 0).sum())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_feature_image: no CUDA device (the numbers are GPU measurements)")
    name, power = _gpu_name_and_power()
    res = run(a.frames, a.device)
    print(json.dumps(dict(metric="feature_image", gpu=name, power_limit=power, frames=a.frames, **res)))


if __name__ == "__main__":
    main()
