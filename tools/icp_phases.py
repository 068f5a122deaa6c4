"""Where the front end's scan match spends its cycles: per-phase clock counts of icp_kernel on bench.py's workload.

    bash tools/build_icp_variants.sh          # scratch/lib_phases.so, built with -DSFE_ICP_PHASE_CLOCKS
    SFE_LIB_PATH=scratch/lib_phases.so python tools/icp_phases.py [--frames 4096] [--steps 3] [--minimizer point]

Runs the same seeded bag and front-end parameters as bench.py (sfe_frontend_run_dev, 20 fixed iterations, window 3)
and prints, from thread 0 of every CTA (icp.cu: ICP_PH_MARK), SM cycles per problem for the set-up and per iteration
for each phase, the ICP stage time by CUDA events, and the CTAs per SM the launch used.  The instrumented build
carries a few extra instructions per phase, so its stage time is a little above the normal build's."""
import argparse
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PHASES = ["set-up (per problem)", "search + re-search list", "trimmed-quantile select", "keep count", "means sums",
          "covariance sums", "fit + end barrier"]
TAU_SOCA = 2.749063720096473


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--minimizer", default="point", choices=["point", "plane"])
    ap.add_argument("--json", default=None, help="also write the table as JSON to this path")
    args = ap.parse_args()
    import torch
    from sonar_slam_b200 import _lib, ops, pipeline, synth
    from sonar_slam_b200.bruce_slam.feature_extraction import FeatureExtraction

    lib = _lib.load()
    if not hasattr(lib, "sfe_icp_phase_clocks"):
        sys.exit(f"{_lib.LIB_PATH} was built without -DSFE_ICP_PHASE_CLOCKS (see tools/build_icp_variants.sh)")
    lib.sfe_icp_phase_clocks.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    lib.sfe_icp_phase_clocks.restype = ctypes.c_int
    buf = (ctypes.c_ulonglong * 17)()

    def clocks(reset):
        if lib.sfe_icp_phase_clocks(buf, 1 if reset else 0) != 0:
            raise RuntimeError("sfe_icp_phase_clocks failed")
        return list(buf)

    torch.cuda.set_device(0)
    F, R = args.frames, 512
    d = synth.make_trajectory_frames(F, seed=0, device="cuda:0")
    fx = FeatureExtraction()
    fx.generate_map_xy(synth.Ping(0, None, 30.0 / R, R, d["bearings"]))
    ctx = ops.context(0)
    maps = _lib.Maps(ctx, fx.map_x, fx.map_y, R, R, fx.width, fx.height)
    mini = 1 if args.minimizer == "plane" else 0
    fe = pipeline.FrontEnd(ctx, maps, max_frames=F, tau=TAU_SOCA,
                           icp=_lib.IcpParams(smooth_length=0, max_iterations=20, minimizer=mini))
    for _ in range(2):
        fe.run_dev(d["frames"].data_ptr(), d["poses_odom"], F)
    clocks(reset=True)
    fe.set_timing(True)
    for _ in range(args.steps):
        fe.run_dev(d["frames"].data_ptr(), d["poses_odom"], F)
    torch.cuda.synchronize()
    stage = fe.get_timing()
    fe.set_timing(False)
    c = clocks(reset=True)
    cyc, cnt, per_sm = c[:7], c[7:14], c[14:17]
    iters = max(cnt[6], 1)
    rows = []
    for k, name in enumerate(PHASES):
        per = cyc[k] / max(cnt[0], 1) if k == 0 else cyc[k] / iters
        rows.append({"phase": name, "cycles": per, "count": cnt[k]})
    total_it = sum(r["cycles"] for r in rows[1:])
    prop = torch.cuda.get_device_properties(0)
    print(f"{prop.name}, {prop.multi_processor_count} SMs; {F} frames x {args.steps} steps, minimizer {args.minimizer}")
    print(f"problems {cnt[0] // args.steps}, iterations {iters // args.steps} per step")
    print(f"{'phase':28s} {'cycles':>10s} {'share of iteration':>20s}")
    for k, r in enumerate(rows):
        share = "" if k == 0 else f"{r['cycles'] / total_it:19.1%}"
        unit = "per problem" if k == 0 else "per iteration"
        print(f"{r['phase']:28s} {r['cycles']:10.0f} {share:>20s}  ({unit})")
    print(f"{'iteration total':28s} {total_it:10.0f}")
    icp_ms = stage["icp"][0] / args.steps
    print(f"ICP stage (CUDA events): {icp_ms:.3f} ms per step")
    print(f"CTAs per SM (128 / 256 / 512-thread launches, 0 = none): {per_sm}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"rows": rows, "iteration_cycles": total_it, "icp_ms_per_step": icp_ms, "ctas_per_sm": per_sm,
                       "gpu": prop.name}, f, indent=1)


if __name__ == "__main__":
    main()
