"""What a SamplingSurfaceNormalDataPointsFilter as the reference's normal source (SFE_ICP_DATA_SAMPLING_NORMALS,
samplingMethod 1, knn 7) costs and saves on the device against the knn normals of a SurfaceNormalDataPointsFilter
(knn 7), point-to-plane, on the workloads of tools/bench_icp_voxel_filter.py.

Workloads:
  map2d     sources of 20 k, 70 k and 200 k points against the 243 726-point map (tools/bench_icp_big_source.py's maps
            and problems), one guess
  wave      the config-3 wave (132-SM-sized batches of 2 000-point sources on 20 000-point targets, 8 waves per call)
  frontend  the batched front end's ICP stage (sfe_frontend_icp_dev) on the frame clouds and window submaps of a
            512-frame bag
Shipped checkers (icp.yaml).  Per row:
  device_ms  the call on device tensors between two CUDA events, median of 5 after a warm-up call (wave: ms per wave)
  stage_ms   torch.profiler kernel time of the data-filter stage of one call, in a separate pass: the compaction pass,
             the sampling-normals kernels, and the CUB sort kernels that start before the call's first map_build or
             ICP kernel (stage_kernels: how many kernels that is)
  kept       the points the filter keeps of the first problem's target
  exact      with the filter, the first three device results equal oracle/sampling_normal_ref.c's bit for bit (status,
             iterations, inliers, T); the knn-normal rows are not checked here (their oracle's brute-force normals
             take hours on the map)
Prints one JSON line with the card's name, power limit and SM clock, read in the same run.

    python tools/bench_icp_sampling_normals.py [--out FILE] [--only map2d:200000]
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))
F32 = np.float32
SN, KNN = 5, 7
STAGE_KERNELS = ("icp_data_filter_kernel", "sn_", "icp_keep_too_large_kernel")
AFTER_FILTERS = ("map_flag_kernel", "icp_kernel", "icp_classify_kernel")


def measure(name, srcs, tgts, guesses, ids, sampling, waves=1, frontend=False):
    """One ops.icp call (or sfe_frontend_icp_dev) over problems p = (srcs[ids[p]], tgts[ids[p]]), point-to-plane with
    knn 7: sampling True takes the normals from the filter, False from the knn search"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    from oracle import oracle as orc
    from oracle import sampling_normal_ref as snr
    from sonar_slam_b200 import _lib, ops

    def pack(cl):
        off = np.zeros(len(cl) + 1, np.int32)
        off[1:] = np.cumsum([len(c) for c in cl])
        return torch.from_numpy(np.concatenate(cl).astype(F32)).cuda(), torch.from_numpy(off).cuda()

    sp, so = pack(srcs)
    tp, to = pack(tgts)
    ii = torch.tensor(ids, dtype=torch.int32).cuda()
    g = torch.from_numpy(np.stack(guesses).astype(F32)).cuda()
    prm = _lib.IcpParams(minimizer=1, normals_knn=KNN)
    chain = dict(reference=[(SN, 1, float("inf"))]) if sampling else None
    flt = _lib.IcpFilters(**chain) if chain else None
    ctx = ops.context(0)
    if frontend:
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
        call = lambda: ops.icp(sp, so, tp, to, g, max(map(len, srcs)), max(map(len, tgts)), prm, src_id=ii,  # noqa
                               tgt_id=ii, filters=flt)
    res = call()
    torch.cuda.synchronize()
    dev = {k: v.cpu().numpy() for k, v in res.items()}
    exact = None
    if sampling:
        exact = True
        for k in range(min(3, len(guesses))):
            w = snr.icp(srcs[ids[k]], tgts[ids[k]], guesses[k], orc.IcpParams(minimizer=1, normals_knn=KNN),
                        snr.IcpFilters(**chain))
            exact &= (int(dev["status"][k]) == w["status"] and int(dev["iterations"][k]) == w["iterations"] and
                      int(dev["inliers"][k]) == w["inliers"] and
                      dev["T"][k].tobytes() == np.asarray(w["T"], F32).tobytes())
    ev = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        torch.cuda.synchronize()
        ev.append(a.elapsed_time(b))
    stage, n_stage = 0.0, 0
    if sampling:
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
    kept = [len(tgts[ids[0]]), len(snr.sampling_normals(tgts[ids[0]], KNN, 1)[0])] if sampling else None
    if frontend:
        _lib.set_icp_filters(ctx, None)
    return dict(name=name, normals="sampling" if sampling else "knn", n_source=len(srcs[ids[0]]),
                n_target=len(tgts[ids[0]]), problems=len(guesses), status=[int(v) for v in dev["status"][:3]],
                iterations=[int(v) for v in dev["iterations"][:3]], device_ms=round(float(np.median(ev)) / waves, 3),
                stage_ms=round(stage / 1e3 / waves, 3), stage_kernels=n_stage, kept=kept, exact=exact)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", default=None, help="the rows whose name:source points starts with this text")
    args = ap.parse_args()
    want = lambda key: args.only is None or key.startswith(args.only)  # noqa: E731
    import torch
    from bench_icp_big_source import maps, problem
    from bench_icp_voxel_filter import card, frontend_problems

    from sonar_slam_b200 import synth
    rows = []
    m2, _ = maps() if want("map2d") else (None, None)
    for n in (20000, 70000, 200000):
        if not want(f"map2d:{n}"):
            continue
        src, gs = problem(m2, n, 1, 8)
        for sampling in (False, True):
            rows.append(measure("map2d", [src], [m2], gs, [0], sampling))
            print(json.dumps(rows[-1]), file=sys.stderr)
    if want("wave"):
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        waves = 8
        pairs = [synth.make_icp_pair(1000 + k, n_source=2000, n_target=20000) for k in range(16)]
        ids = [k % 16 for k in range(sms * waves)]
        for sampling in (False, True):
            rows.append(measure("wave", [p[0] for p in pairs], [p[1] for p in pairs],
                                [pairs[i][2].astype(F32) for i in ids], ids, sampling, waves=waves))
            print(json.dumps(rows[-1]), file=sys.stderr)
    if want("frontend"):
        srcs, tgts, gs = frontend_problems(512)
        ids = list(range(len(gs)))
        for sampling in (False, True):
            rows.append(measure("frontend", srcs, tgts, gs, ids, sampling, frontend=True))
            print(json.dumps(rows[-1]), file=sys.stderr)
    name, power, clock = card()
    line = json.dumps(dict(gpu=name, power_limit=power, sm_clock_max=clock, checkers="shipped", rows=rows))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
