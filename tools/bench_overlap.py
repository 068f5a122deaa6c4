"""Schedule of the resident-frame front end (sfe_frontend_run_dev): the serial schedule (every stage over the whole
batch, one after another) against the overlapped one (feature stages of one sub-batch next to the scan matching of the
previous one, on two streams; sfe_frontend_set_overlap), on bench.py's workload.  Prints one JSON line and writes
nothing.
Run on an H100:  PYTHONPATH=. python tools/bench_overlap.py [--frames F] [--steps K] [--reps N] [--subs 256,512,1024]

  ms_per_step[schedule]   CUDA events around K back-to-back run_dev calls / K; `reps` measurements per schedule, the
                          schedules alternated within every repetition (median, min, max)
  priority[order]         the default sub-batch with the match stream first (default), the feature stream first, or
                          equal priorities (SFE_FE_OVERLAP_PRIO, one front end each, alternated the same way)
  sliced[S]               the serial schedule fed S frames per call (window carried across calls): what the stages
                          cost at the sub-batch size alone, without the overlap -- ms per F frames, and per stage
                          (per-stage CUDA events, sfe_frontend_set_timing)
  enqueue_ms[schedule]    host time of one run_dev call (it returns before the GPU is done), median over `reps` calls
                          made after a device sync; it must stay below the GPU step for the GPU to stay fed
  identical               every schedule left bit-identical T, iterations, inliers, status and clouds on the device
"""
import argparse
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

TAU_SOCA = 2.749063720096473
R = B = 512


def _stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--subs", default="256,512,1024")
    args = ap.parse_args()
    import torch
    from bench import gpu_info
    from sonar_slam_b200 import _lib, ops, pipeline, synth
    from sonar_slam_b200.bruce_slam.feature_extraction import FeatureExtraction

    F, K = args.frames, args.steps
    subs = [int(s) for s in args.subs.split(",")]
    torch.cuda.set_device(0)
    d = synth.make_trajectory_frames(F, seed=0, device="cuda:0")   # bench.py's bag replay
    frames, poses = d["frames"], d["poses_odom"]
    fx = FeatureExtraction()
    fx.generate_map_xy(synth.Ping(0, None, 30.0 / R, R, d["bearings"]))
    ctx = ops.context(0)
    maps = _lib.Maps(ctx, fx.map_x, fx.map_y, R, B, fx.width, fx.height)

    def front_end():
        return pipeline.FrontEnd(ctx, maps, max_frames=F, tau=TAU_SOCA,
                                 icp=_lib.IcpParams(smooth_length=0, max_iterations=20))

    def step_ms(fe, sub):
        fe.set_overlap(sub)
        fe.run_dev(frames.data_ptr(), poses, F)                       # (schedule switch: not timed)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(K):
            fe.run_dev(frames.data_ptr(), poses, F)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / K

    def outputs(fe):
        r = fe.results_dev()
        out = [ctx.to_host(r["T"], (F, 9), np.float32).view(np.uint32)]
        out += [ctx.to_host(r[k], (F,), np.int32) for k in ("iterations", "inliers", "status", "cloud_count")]
        xy = ctx.to_host(r["cloud_xy"], (F, r["cloud_stride"], 2), np.float32).view(np.uint32)
        out += [xy[i, :c] for i, c in enumerate(out[-1])]
        return out

    def same(a, b):
        return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))

    # ---- schedules, alternated
    fe = front_end()
    scheds = [0] + subs
    ref, identical = None, {}
    for s in scheds:                                                  # warm-up (and the outputs of every schedule)
        step_ms(fe, s)
        o = outputs(fe)
        ref = o if s == 0 else ref
        identical[str(s)] = same(o, ref)
    ms = {str(s): [] for s in scheds}
    for _ in range(args.reps):
        for s in scheds:
            ms[str(s)].append(step_ms(fe, s))

    def sliced_ms(fe, sub):
        fe.set_overlap(0)
        fe.set_carry(True)

        def step():
            for f0 in range(0, F, sub):
                n = min(sub, F - f0)
                fe.run_dev(frames[f0:].data_ptr(), poses[f0:f0 + n], n)
        step()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(K):
            step()
        e1.record()
        torch.cuda.synchronize()
        fe.set_timing(True)
        for _ in range(K):
            step()
        stages = {k: v[0] / K for k, v in fe.get_timing().items()}
        fe.set_timing(False)
        fe.set_carry(False)
        return {"ms_per_step": e0.elapsed_time(e1) / K, "stage_ms_per_step": stages}
    sliced = {str(s): sliced_ms(fe, s) for s in [F] + subs}
    enq = {}
    for s in (0, subs[len(subs) // 2]):
        fe.set_overlap(s)
        ts = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fe.run_dev(frames.data_ptr(), poses, F)
            ts.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()
        enq[str(s)] = _stats(ts)
    fe.close()

    # ---- stream priorities at the middle sub-batch, one front end per order (read when it is created)
    sub = subs[len(subs) // 2]
    fes = {}
    for order in ("match", "features", "equal"):
        os.environ["SFE_FE_OVERLAP_PRIO"] = order
        fes[order] = front_end()
    os.environ.pop("SFE_FE_OVERLAP_PRIO")
    prio = {k: [] for k in fes}
    for k, f in fes.items():
        step_ms(f, sub)
        identical[f"{sub}/{k}"] = same(outputs(f), ref)
    for _ in range(args.reps):
        for k, f in fes.items():
            prio[k].append(step_ms(f, sub))
    for f in fes.values():
        f.close()

    serial = float(np.median(ms["0"]))
    line = {"gpu": gpu_info(0), "frames": F, "steps_per_measurement": K, "reps": args.reps,
            "ms_per_step": {k: _stats(v) for k, v in ms.items()},
            "frames_per_s": {k: F / (float(np.median(v)) * 1e-3) for k, v in ms.items()},
            "speedup_vs_serial": {k: serial / float(np.median(v)) for k, v in ms.items()},
            "priority_sub_batch": sub, "priority": {k: _stats(v) for k, v in prio.items()},
            "sliced": sliced, "enqueue_ms": enq, "identical": identical}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
