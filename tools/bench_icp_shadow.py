"""What a reading SurfaceNormalDataPointsFilter with a ShadowDataPointsFilter after it (SFE_ICP_DATA_NORMALS knn 5,
SFE_ICP_DATA_SHADOW eps 0.1) costs on the device, against the same ICP call without the reading chain, point-to-point
with the shipped checkers.

Workloads:
  wave      the config-3 wave (132-SM-sized batches of 2 000-point sources on 20 000-point targets, 8 waves per call)
  frontend  the batched front end's ICP stage (sfe_frontend_icp_dev) on the frame clouds and window submaps of a
            512-frame bag
  map2d     sources of 20 k and 200 k points against the 243 726-point map (tools/bench_icp_big_source.py's maps and
            problems), one guess
Per row:
  device_ms  the call on device tensors between two CUDA events, median of 5 after a warm-up call (wave: ms per wave)
  stage_ms   torch.profiler kernel time of the reading chain of one call, in a separate pass: the compaction and
             shadow passes (icp_data_filter_kernel), the normals kernels (snrm_*) and, for clouds above 4 096 points,
             the map_build kernels and sorts between snrm_counts_kernel and snrm_scatter_kernel (stage_kernels: the
             names of those kernels, with their counts)
  kept       the points the chain keeps of the first problem's source
  exact      the first three device results equal the oracle's bit for bit (status, iterations, inliers, T):
             oracle/shadow_ref.c with the chain, oracle/oracle.py without it
Prints one JSON line with the card's name, power limit and SM clock, read in the same run.

    python tools/bench_icp_shadow.py [--out FILE] [--only map2d:200000]
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
KNN, EPS = 5, 0.1
CHAIN = [(6, KNN, 0.0), (7, 0, EPS)]  # _lib.NORMALS, _lib.SHADOW


def measure(name, srcs, tgts, guesses, ids, shadow, waves=1, frontend=False):
    """One ops.icp call (or sfe_frontend_icp_dev) over problems p = (srcs[ids[p]], tgts[ids[p]]), with (shadow True)
    or without the reading chain"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    from oracle import oracle as orc
    from oracle import shadow_ref as shr
    from sonar_slam_b200 import _lib, ops

    def pack(cl):
        off = np.zeros(len(cl) + 1, np.int32)
        off[1:] = np.cumsum([len(c) for c in cl])
        return torch.from_numpy(np.concatenate(cl).astype(F32)).cuda(), torch.from_numpy(off).cuda()

    sp, so = pack(srcs)
    tp, to = pack(tgts)
    ii = torch.tensor(ids, dtype=torch.int32).cuda()
    g = torch.from_numpy(np.stack(guesses).astype(F32)).cuda()
    prm = _lib.IcpParams()
    flt = _lib.IcpFilters(reading=CHAIN) if shadow else None
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
    exact = True
    for k in range(min(3, len(guesses))):
        s, t = srcs[ids[k]], tgts[ids[k]]
        w = shr.icp(s, t, guesses[k], orc.IcpParams(), shr.IcpFilters(reading=CHAIN)) if shadow else \
            orc.icp(s, t, guesses[k], orc.IcpParams())
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
    stage, n_stage = 0.0, {}
    if shadow:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        kern = [e for e in prof.events() if e.device_type.name == "CUDA" and "memcpy" not in e.name.lower() and
                "memset" not in e.name.lower()]
        mark = [e.time_range.start for e in kern if "snrm_counts_kernel" in e.name or "snrm_scatter_kernel" in e.name]
        names = {}
        for e in kern:
            if ("icp_data_filter_kernel" in e.name or "snrm_" in e.name or
                    (len(mark) == 2 and mark[0] < e.time_range.start < mark[1])):
                us = getattr(e, "device_time_total", None)
                stage += us if us is not None else e.cuda_time_total
                key = e.name.split("(")[0].replace("void ", "")[:60]
                names[key] = names.get(key, 0) + 1
        n_stage = names
    kept = [len(srcs[ids[0]]), len(shr.data_filters(srcs[ids[0]], CHAIN))] if shadow else None
    if frontend:
        _lib.set_icp_filters(ctx, None)
    return dict(name=name, chain="normals+shadow" if shadow else "none", n_source=len(srcs[ids[0]]),
                n_target=len(tgts[ids[0]]), problems=len(guesses), status=[int(v) for v in dev["status"][:3]],
                iterations=[int(v) for v in dev["iterations"][:3]], device_ms=round(float(np.median(ev)) / waves, 3),
                stage_ms=round(stage / 1e3 / waves, 3), stage_kernels=n_stage, kept=kept, exact=bool(exact))


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
    if want("wave"):
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        waves = 8
        pairs = [synth.make_icp_pair(1000 + k, n_source=2000, n_target=20000) for k in range(16)]
        ids = [k % 16 for k in range(sms * waves)]
        for shadow in (False, True):
            rows.append(measure("wave", [p[0] for p in pairs], [p[1] for p in pairs],
                                [pairs[i][2].astype(F32) for i in ids], ids, shadow, waves=waves))
            print(json.dumps(rows[-1]), file=sys.stderr)
    if want("frontend"):
        srcs, tgts, gs = frontend_problems(512)
        ids = list(range(len(gs)))
        for shadow in (False, True):
            rows.append(measure("frontend", srcs, tgts, gs, ids, shadow, frontend=True))
            print(json.dumps(rows[-1]), file=sys.stderr)
    m2, _ = maps() if want("map2d") else (None, None)
    for n in (20000, 200000):
        if not want(f"map2d:{n}"):
            continue
        src, gs = problem(m2, n, 1, 8)
        for shadow in (False, True):
            rows.append(measure("map2d", [src], [m2], gs, [0], shadow))
            print(json.dumps(rows[-1]), file=sys.stderr)
    name, power, clock = card()
    line = json.dumps(dict(gpu=name, power_limit=power, sm_clock_max=clock, checkers="shipped", rows=rows))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
