"""Where the front end's frame down-sample spends its cycles: per-phase clock counts of the down-sample kernels on
bench.py's workload.

    bash tools/build_ds_variants.sh           # scratch/lib_dsphases.so, built with -DSFE_DS_PHASE_CLOCKS
    SFE_LIB_PATH=scratch/lib_dsphases.so python tools/ds_phases.py [--frames 4096] [--steps 3]

Runs the same seeded bag and front-end parameters as bench.py (sfe_frontend_run_dev) and prints, from thread 0 of
every CTA (cloud.cu: DS_PH_MARK), SM cycles per cloud for each phase, the down-sample stage time by CUDA events, and
the CTAs per SM of the last launch.  The window submaps' down-sample runs the same kernel and would add its clouds
to the same counters, so the submap thinning is switched off here (submap_resolution = 0; ICP then matches unthinned
targets, which does not touch the frame filters)."""
import argparse
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PHASES = ["bounds", "keys + sort by cell", "rank in cell / leaf heads", "medoid sums", "leaf emit"]
TAU_SOCA = 2.749063720096473


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the table as JSON to this path")
    args = ap.parse_args()
    import torch
    from sonar_slam_b200 import _lib, ops, pipeline, synth
    from sonar_slam_b200.bruce_slam.feature_extraction import FeatureExtraction

    lib = _lib.load()
    if not hasattr(lib, "sfe_ds_phase_clocks"):
        sys.exit(f"{_lib.LIB_PATH} was built without -DSFE_DS_PHASE_CLOCKS (see tools/build_ds_variants.sh)")
    lib.sfe_ds_phase_clocks.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
    lib.sfe_ds_phase_clocks.restype = ctypes.c_int
    buf = (ctypes.c_ulonglong * 11)()

    def clocks(reset):
        if lib.sfe_ds_phase_clocks(buf, 1 if reset else 0) != 0:
            raise RuntimeError("sfe_ds_phase_clocks failed")
        return list(buf)

    torch.cuda.set_device(0)
    F, R = args.frames, 512
    d = synth.make_trajectory_frames(F, seed=0, device="cuda:0")
    fx = FeatureExtraction()
    fx.generate_map_xy(synth.Ping(0, None, 30.0 / R, R, d["bearings"]))
    ctx = ops.context(0)
    maps = _lib.Maps(ctx, fx.map_x, fx.map_y, R, R, fx.width, fx.height)
    fe = pipeline.FrontEnd(ctx, maps, max_frames=F, tau=TAU_SOCA, submap_resolution=0.0,
                           icp=_lib.IcpParams(smooth_length=0, max_iterations=20))
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
    cyc, cnt, per_sm = c[:5], c[5:10], c[10]
    clouds = max(cnt[0], 1)
    rows = [{"phase": name, "cycles": cyc[k] / clouds, "count": cnt[k]} for k, name in enumerate(PHASES)]
    total = sum(r["cycles"] for r in rows)
    prop = torch.cuda.get_device_properties(0)
    print(f"{prop.name}, {prop.multi_processor_count} SMs; {F} frames x {args.steps} steps")
    print(f"clouds {cnt[0] // args.steps} per step")
    print(f"{'phase':28s} {'cycles per cloud':>17s} {'share':>8s}")
    for r in rows:
        print(f"{r['phase']:28s} {r['cycles']:17.0f} {r['cycles'] / max(total, 1):8.1%}")
    print(f"{'total':28s} {total:17.0f}")
    ds_ms = stage["downsample"][0] / args.steps
    print(f"downsample stage (CUDA events): {ds_ms:.3f} ms per step")
    print(f"CTAs per SM of the last launch: {per_sm}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"rows": rows, "cloud_cycles": total, "downsample_ms_per_step": ds_ms, "ctas_per_sm": per_sm,
                       "gpu": prop.name}, f, indent=1)


if __name__ == "__main__":
    main()
