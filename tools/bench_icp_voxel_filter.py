"""What a VoxelGridDataPointsFilter in the ICP chain (SFE_ICP_DATA_VOXEL) costs and saves on the device, on the
workloads of tools/bench_icp_octree_filter.py so that the two down-samplers compare row for row.

Workloads:
  map2d     the README's 2-D map-to-map rows: sources of 20 k, 70 k and 200 k points against the 243 726-point map
            (tools/bench_icp_big_source.py's maps and problems), 1 and 30 guesses; without a filter, and with a
            reading voxel filter of vSize 0.2 m and 0.5 m
  wave      the config-3 wave (132-SM-sized batches of 2 000-point sources on 20 000-point targets, 8 waves per call)
            without a filter and with a reference voxel filter of 0.2 m
  frontend  the batched front end's ICP stage (sfe_frontend_icp_dev) on the frame clouds and window submaps of a
            512-frame bag, without a filter and with a 0.2 m voxel filter on both clouds
Shipped checkers (icp.yaml).  Per row:
  device_ms  the call on device tensors between two CUDA events, median of 5 after a warm-up call (wave: ms per wave)
  voxel_ms   torch.profiler kernel time of the data-filter stage of one call, in a separate pass: the compaction pass,
             the voxel kernels and the size restore, with the CUB sort and scan kernels that start before the call's
             first map_build or ICP kernel (stage_kernels: how many kernels that is)
  kept       the points the filter keeps of the first problem's filtered cloud
  exact      the first three device results equal oracle/voxel_filter_ref.c's bit for bit (status, iterations,
             inliers, T)
Prints one JSON line with the card's name, power limit and SM clock, read in the same run.

    python tools/bench_icp_voxel_filter.py [--out FILE] [--only map2d:200000]
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
sys.path.insert(0, os.path.join(REPO, "tools"))
F32 = np.float32
VOX = 4
# the data-filter stage's own kernels; CUB's sort and scan count too when they start before the call's first
# map_build or ICP kernel (map_build sorts with CUB as well)
STAGE_KERNELS = ("icp_data_filter_kernel", "vox_", "dsg_bounds_kernel", "icp_keep_too_large_kernel")
AFTER_FILTERS = ("map_flag_kernel", "icp_kernel", "icp_classify_kernel")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [x.strip() for x in q.split(",")]
    except Exception:  # noqa: BLE001
        import torch
        return torch.cuda.get_device_name(0), "unknown", "unknown"


def measure(name, srcs, tgts, guesses, src_id, tgt_id, filters, waves=1, frontend=False):
    """One ops.icp call over P = len(guesses) problems; problem p: srcs[src_id[p]] onto tgts[tgt_id[p]].  frontend:
    sfe_frontend_icp_dev on problem p = (srcs[p], tgts[p]) instead, the filters set on the context."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    import ctypes

    from oracle import oracle as orc
    from oracle import voxel_filter_ref as vfr
    from sonar_slam_b200 import _lib, ops

    def pack(cl):
        off = np.zeros(len(cl) + 1, np.int32)
        off[1:] = np.cumsum([len(c) for c in cl])
        return torch.from_numpy(np.concatenate(cl).astype(F32)).cuda(), torch.from_numpy(off).cuda()

    sp, so = pack(srcs)
    tp, to = pack(tgts)
    si = torch.tensor(src_id, dtype=torch.int32).cuda()
    ti = torch.tensor(tgt_id, dtype=torch.int32).cuda()
    g = torch.from_numpy(np.stack(guesses).astype(F32)).cuda()
    prm = _lib.IcpParams()
    flt = _lib.IcpFilters(**filters) if filters else None
    if frontend:
        ctx = ops.context(0)
        P = len(guesses)
        T = torch.empty((P, 3, 3), dtype=torch.float32, device="cuda")
        iters, inl, st = (torch.empty(P, dtype=torch.int32, device="cuda") for _ in range(3))
        p_ = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731

        def call():
            _lib.set_icp_filters(ctx, flt)
            _lib.check(ctx.lib.sfe_frontend_icp_dev(ctx.handle, ctypes.byref(prm), p_(sp), p_(so), p_(tp), p_(to), P,
                                                    max(map(len, srcs)), max(map(len, tgts)), p_(g), p_(T),
                                                    p_(iters), p_(inl), p_(st), None), "sfe_frontend_icp_dev")
            return dict(T=T, iterations=iters, inliers=inl, status=st)
    else:
        call = lambda: ops.icp(sp, so, tp, to, g, max(map(len, srcs)), max(map(len, tgts)), prm, src_id=si,
                               tgt_id=ti, filters=flt)
    res = call()
    torch.cuda.synchronize()
    dev = {k: v.cpu().numpy() for k, v in res.items()}
    oflt = vfr.IcpFilters(**filters) if filters else vfr.IcpFilters()
    exact = True
    for k in range(min(3, len(guesses))):
        w = vfr.icp(srcs[src_id[k]], tgts[tgt_id[k]], guesses[k], orc.IcpParams(), oflt)
        exact &= (int(dev["status"][k]) == w["status"] and int(dev["iterations"][k]) == w["iterations"] and
                  int(dev["inliers"][k]) == w["inliers"] and dev["T"][k].tobytes() == np.asarray(w["T"], F32).tobytes())
    ev = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        torch.cuda.synchronize()
        ev.append(a.elapsed_time(b))
    stage, n_stage = 0.0, 0
    if filters:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        kern = [e for e in prof.events() if e.device_type.name == "CUDA" and "memcpy" not in e.name.lower() and
                "memset" not in e.name.lower()]
        end = min([e.time_range.start for e in kern if any(k in e.name for k in AFTER_FILTERS)], default=float("inf"))
        for e in kern:
            if any(k in e.name for k in STAGE_KERNELS) or ("cub" in e.name.lower() and e.time_range.start < end):
                us = getattr(e, "device_time_total", None)
                stage += us if us is not None else e.cuda_time_total
                n_stage += 1
    kept = None
    if filters:
        side = "reading" if filters.get("reading") else "reference"
        cloud = srcs[src_id[0]] if side == "reading" else tgts[tgt_id[0]]
        kept = [side, len(cloud), len(vfr.data_filters(cloud, filters[side]))]
    return dict(name=name, filters=filters, n_source=len(srcs[src_id[0]]), n_target=len(tgts[tgt_id[0]]),
                problems=len(guesses), status=[int(v) for v in dev["status"][:3]],
                iterations=[int(v) for v in dev["iterations"][:3]], device_ms=round(float(np.median(ev)) / waves, 3),
                voxel_ms=round(stage / 1e3 / waves, 3), stage_kernels=n_stage, kept=kept, exact=bool(exact))


def frontend_problems(n_frames):
    """The front end's scan-match problems of an n_frames bag: every frame's cloud (reading) against the window
    submap before it (reference), from the guess odometry gives, as oracle/pipeline_ref builds them."""
    from oracle import featx_ref
    from oracle import oracle as orc
    from oracle import pipeline_ref as pr
    from sonar_slam_b200 import synth
    d = synth.make_trajectory_frames(n_frames, seed=1)
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    poses = d["poses_odom"]
    clouds = [pr.slam_cloud(pr.frame_cloud(f, geo)) for f in d["frames"].numpy()]
    srcs, tgts, gs = [], [], []
    for i in range(1, len(clouds)):
        parts = [pr.transform_points(clouds[k], pr.between(poses[i - 1], poses[k])) for k in range(max(0, i - 3), i)]
        tgt = orc.downsample(np.concatenate(parts), 0.5)[0]
        if len(clouds[i]) >= 30 and len(tgt) >= 30:
            srcs.append(clouds[i]), tgts.append(tgt), gs.append(pr.between(poses[i - 1], poses[i]))
    return srcs, tgts, gs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", default=None, help="the rows whose name:source points starts with this text")
    args = ap.parse_args()
    want = lambda key: args.only is None or key.startswith(args.only)
    import torch
    from bench_icp_big_source import maps, problem

    from sonar_slam_b200 import synth
    rows = []
    m2, _ = maps() if want("map2d") else (None, None)
    for n in (20000, 70000, 200000):
        if not want(f"map2d:{n}"):
            continue
        for k in (1, 30):
            src, gs = problem(m2, n, k, 8)
            chains = [None] + [dict(reading=[(VOX, 1, size)]) for size in (0.2, 0.5)]
            for ch in chains:
                rows.append(measure("map2d", [src], [m2], gs, [0] * k, [0] * k, ch))
                print(json.dumps(rows[-1]), file=sys.stderr)
    if want("wave"):
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        waves = 8
        P = sms * waves
        pairs = [synth.make_icp_pair(1000 + k, n_source=2000, n_target=20000) for k in range(16)]
        ids = [k % 16 for k in range(P)]
        gs = [pairs[i][2].astype(F32) for i in ids]
        for ch in [None, dict(reference=[(VOX, 1, 0.2)])]:
            rows.append(measure("wave", [p[0] for p in pairs], [p[1] for p in pairs], gs, ids, ids, ch, waves=waves))
            print(json.dumps(rows[-1]), file=sys.stderr)
    if want("frontend"):
        srcs, tgts, gs = frontend_problems(512)
        ids = list(range(len(gs)))
        for ch in [None, dict(reading=[(VOX, 1, 0.2)], reference=[(VOX, 1, 0.2)])]:
            rows.append(measure("frontend", srcs, tgts, gs, ids, ids, ch, frontend=True))
            print(json.dumps(rows[-1]), file=sys.stderr)
    name, power, clock = card()
    line = json.dumps(dict(gpu=name, power_limit=power, sm_clock_max=clock, checkers="shipped", rows=rows))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
