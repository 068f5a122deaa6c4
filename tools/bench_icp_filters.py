"""What the ICP filters (sfe_icp_filters) cost on the device.

  1. config-3 scan matches (2 000-point sources on 20 000-point targets, bench.py's loop-closure shape): one wave = one
     problem per SM, 8 waves per call; ms per wave for the shipped chain, + MedianDistOutlierFilter (a second exact
     selection per iteration), + data filters (the compaction pass before the launch), and everything together;
  2. the batched front end's ICP stage (sfe_frontend_set_timing) on a synthetic bag, with and without the filters.

    python tools/bench_icp_filters.py [--frames 512] [--reps 5]

Prints one JSON line with the card's name and power limit beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sonar_slam_b200 import _lib, ops, pipeline, synth  # noqa: E402

MX, MN = _lib.MAX_DIST, _lib.MIN_DIST
CHAINS = {
    "shipped": None,
    "median": dict(median_factor=3.0),
    "data_filters": dict(reading=[(MN, -1, 1.0), (MX, -1, 28.0)], reference=[(MX, -1, 40.0)]),
    "all": dict(min_dist=0.01, median_factor=3.0, reading=[(MN, -1, 1.0), (MX, -1, 28.0)],
                reference=[(MX, -1, 40.0)]),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def time_call(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), float(min(ts))


def config3(ctx, reps, waves=8):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    P = sms * waves
    pairs = [synth.make_icp_pair(1000 + k % 16, n_source=2000, n_target=20000) for k in range(16)]
    srcs = [pairs[k % 16][0] for k in range(P)]
    tgts = [pairs[k % 16][1] for k in range(P)]

    def pack(cl):
        off = np.zeros(len(cl) + 1, np.int32)
        off[1:] = np.cumsum([len(c) for c in cl])
        return torch.from_numpy(np.concatenate(cl)).cuda(), torch.from_numpy(off).cuda()

    sp, so = pack(srcs)
    tp, to = pack(tgts)
    g = torch.from_numpy(np.stack([pairs[k % 16][2] for k in range(P)]).astype(np.float32)).cuda()
    ns, nt = max(map(len, srcs)), max(map(len, tgts))
    out = {}
    for name, kw in CHAINS.items():
        flt = _lib.IcpFilters(**kw) if kw else None
        med, best = time_call(lambda: ops.icp(sp, so, tp, to, g, ns, nt, _lib.IcpParams(), ctx=ctx, filters=flt), reps)
        out[name] = dict(ms_per_wave=round(med / waves, 4), ms_per_wave_min=round(best / waves, 4))
    return dict(problems=P, waves=waves, chains=out)


def frontend(ctx, frames, reps):
    d = synth.make_trajectory_frames(frames, seed=5)
    from oracle import featx_ref
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    dev = d["frames"].cuda()
    out = {}
    for name in ("shipped", "all"):
        kw = CHAINS[name]
        fe = pipeline.FrontEnd(ctx, maps, max_frames=frames, icp_filters=_lib.IcpFilters(**kw) if kw else None)
        for _ in range(2):
            fe.run_dev(dev.data_ptr(), d["poses_odom"], frames)
        ctx.sync()
        fe.set_timing(True)
        fe.get_timing()
        for _ in range(reps):
            fe.run_dev(dev.data_ptr(), d["poses_odom"], frames)
        ctx.sync()
        ms, calls = fe.get_timing()["icp"]
        out[name] = dict(icp_stage_ms_per_call=round(ms / max(reps, 1), 4), timed_intervals=int(calls))
        fe.close()
    return dict(frames=frames, chains=out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    ctx = ops.context(0)
    name, power = card()
    res = dict(gpu=name, power_limit=power, config3=config3(ctx, a.reps), frontend=frontend(ctx, a.frames, a.reps))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
