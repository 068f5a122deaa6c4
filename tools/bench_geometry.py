"""Cost of per-frame sonar geometry in the resident-frame front end (sfe_frontend_run_dev_geometry): bench.py's bag
replay rendered under two geometries -- 512 x 512 at 30 m (geometry 0, the slots) and 384 x 512 at 20 m (geometry 1) --
and fed as one batch with the geometry switching never, once in the middle, or every 64 frames.  Every switch adds a
CFAR and a Cartesian-point launch (and, for geometry 1, a copy that packs the run at its natural stride); the stages
after the Cartesian points stay one launch each.  Prints one JSON line and writes nothing.
Run on an H100:  PYTHONPATH=. python tools/bench_geometry.py [--frames F] [--steps K] [--reps N]

  ms_per_step[bag]        CUDA events around K back-to-back run_dev calls / K; `reps` measurements per bag, the bags
                          alternated within every repetition (median, min, max)
  stage_ms_per_step[bag]  per-stage CUDA events (sfe_frontend_set_timing) over K further calls / K, with the number of
                          timed intervals per call (CFAR and Cartesian points: one per run of one geometry)
  bags: plain (sfe_frontend_run_dev, geometry 0), g0 / g1 (every frame in geometry 0 / 1 through the geometry entry
  point), switch_mid (geometry 0 then 1), switch_64 (0 and 1 alternating every 64 frames)
"""
import argparse
import json
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

TAU_SOCA = 2.749063720096473
SHAPES = [(512, 512, 30.0), (384, 512, 20.0)]


def _stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import torch
    from bench import gpu_info
    from sonar_slam_b200 import _lib, ops, pipeline, synth
    from sonar_slam_b200.bruce_slam.feature_extraction import FeatureExtraction

    F, K = args.frames, args.steps
    torch.cuda.set_device(0)
    ctx = ops.context(0)
    rendered, maps = [], []
    for R, B, rmax in SHAPES:
        d = synth.make_trajectory_frames(F, seed=0, num_ranges=R, num_beams=B, max_range=rmax, device="cuda:0")
        fx = FeatureExtraction()
        fx.generate_map_xy(synth.Ping(0, None, rmax / R, R, d["bearings"]))
        maps.append(_lib.Maps(ctx, fx.map_x, fx.map_y, R, B, fx.width, fx.height))
        rendered.append(d["frames"].reshape(F, -1))
        poses = d["poses_odom"]
    idx = np.arange(F)
    schedules = {"g0": np.zeros(F, np.int32), "g1": np.ones(F, np.int32),
                 "switch_mid": (idx >= F // 2).astype(np.int32), "switch_64": ((idx // 64) % 2).astype(np.int32)}
    slots = {}
    for name, g in schedules.items():   # frame i of geometry g in the first R_g * B_g bytes of its 512 x 512 slot
        s = torch.zeros((F, 512 * 512), dtype=torch.uint8, device="cuda:0")
        for k in (0, 1):
            sel = torch.from_numpy(np.flatnonzero(g == k)).cuda()
            s[sel, :rendered[k].shape[1]] = rendered[k][sel]
        slots[name] = s
    fe = pipeline.FrontEnd(ctx, maps[0], max_frames=F, tau=TAU_SOCA, icp=_lib.IcpParams(smooth_length=0,
                                                                                       max_iterations=20))
    assert fe.add_geometry(maps[1]) == 1

    def call(name):
        if name == "plain":
            fe.run_dev(slots["g0"].data_ptr(), poses, F)
        else:
            fe.run_dev(slots[name].data_ptr(), poses, F, geometry=schedules[name])

    def step_ms(name):
        call(name)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(K):
            call(name)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / K

    bags = ["plain"] + list(schedules)
    matched = {}
    for b in bags:                      # warm-up, and how many frames each bag matches
        step_ms(b)
        r = fe.results_dev()
        matched[b] = int((ctx.to_host(r["status"], (F,), np.int32) == 0).sum())
    ms = {b: [] for b in bags}
    for _ in range(args.reps):
        for b in bags:
            ms[b].append(step_ms(b))
    stages = {}
    for b in bags:
        fe.set_timing(True)
        for _ in range(K):
            call(b)
        stages[b] = {k: {"ms": v[0] / K, "intervals": v[1] / K} for k, v in fe.get_timing().items()}
        fe.set_timing(False)
    fe.close()
    line = {"gpu": gpu_info(0), "frames": F, "steps_per_measurement": K, "reps": args.reps,
            "runs": {k: 1 + int((np.diff(g) != 0).sum()) for k, g in schedules.items()},
            "ms_per_step": {k: _stats(v) for k, v in ms.items()},
            "frames_per_s": {k: F / (float(np.median(v)) * 1e-3) for k, v in ms.items()},
            "stage_ms_per_step": stages, "frames_matched": matched}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
