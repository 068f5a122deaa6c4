"""3-D scan matching on the device (`ops.icp` / `pcl.ICP` on [N,3] clouds), every row checked bit for bit against
oracle/icp3_ref.c.

    python tools/bench_icp_3d.py [--pairs 132] [--reps 5] [--out FILE]

Rows:
  config3      one wave of 2 000 x 20 000-point 3-D config-3 pairs (synth.make_icp_pair3), fixed 20 iterations and the
               shipped checkers, CUDA events around ops.icp; next to it the 2-D path on the same clouds' x, y columns
  closure      loop-closure-shaped calls: a 1 500-point source, 30 guesses, 25 k / 100 k / 250 k-point targets; the map
               grid build (map_* kernels, CUB's sort and scan, icp3_map_z_kernel) and the ICP kernel separated with
               torch.profiler, the whole call by CUDA events
  compute_batch  pcl.ICP.compute_batch end to end (host arrays in and out), host clock
  oracle       the CPU oracle on one host thread, per problem
The card's name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import icp3_ref as o3, oracle as orc  # noqa: E402
from sonar_slam_b200 import _lib, ops, synth  # noqa: E402
from sonar_slam_b200.bruce_slam import pcl  # noqa: E402

FIXED20 = dict(max_iterations=20, smooth_length=0)


def packed(clouds):
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    return torch.from_numpy(np.ascontiguousarray(np.concatenate(clouds))).cuda(), torch.from_numpy(off).cuda()


def events(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), out


def exact(out, want):
    T, st, it, inl = (out[k].cpu().numpy() if torch.is_tensor(out[k]) else out[k]
                      for k in ("T", "status", "iterations", "inliers"))
    return all(st[p] == w["status"] and it[p] == w["iterations"] and inl[p] == w["inliers"] and
               T[p].tobytes() == np.float32(w["T"]).tobytes() for p, w in enumerate(want))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=132)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the rows as JSON to FILE")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_icp_3d needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    rows = []
    ctx = ops.context(0)

    # ---- config-3 waves, 3-D and the 2-D path on the same x, y
    pairs = [synth.make_icp_pair3(2000 + k) for k in range(a.pairs)]
    srcs, tgts = [p[0] for p in pairs], [p[1] for p in pairs]
    sp3, so = packed(srcs)
    tp3, to = packed(tgts)
    sp2, tp2 = sp3[:, :2].contiguous(), tp3[:, :2].contiguous()
    g3 = torch.eye(4).repeat(a.pairs, 1, 1).cuda()
    g2 = torch.eye(3).repeat(a.pairs, 1, 1).cuda()
    for name, prm in (("fixed20", FIXED20), ("shipped", {})):
        p = _lib.IcpParams(**prm)
        t3, out3 = events(lambda: ops.icp(sp3, so, tp3, to, g3, 2000, 20000, p, ctx=ctx), a.reps)
        t2, _ = events(lambda: ops.icp(sp2, so, tp2, to, g2, 2000, 20000, p, ctx=ctx), a.reps)
        want = o3.icp3_many([(s, t, np.eye(4, dtype=np.float32)) for s, t in zip(srcs, tgts)], orc.IcpParams(**prm))
        rows.append(dict(row="config3", checkers=name, problems=a.pairs, ms_3d=t3, ms_2d_same_xy=t2,
                         mean_iterations_3d=float(out3["iterations"].float().mean()), exact=exact(out3, want)))

    # ---- loop-closure-shaped calls
    rng = np.random.default_rng(1)
    for n_target in (25_000, 100_000, 250_000):
        src, tgt, _ = synth.make_icp_pair3(5, n_source=1500, n_target=n_target, extent=60.0 * max(1.0, np.sqrt(n_target / 40000)))
        guesses = np.stack([np.eye(4, dtype=np.float32)] + [
            synth.se3(rng.uniform(-0.3, 0.3, 3), rng.normal(size=3), rng.uniform(-0.05, 0.05)).astype(np.float32)
            for _ in range(29)])
        sp, so1 = packed([src])
        tp, to1 = packed([tgt])
        g = torch.from_numpy(guesses).cuda()
        ids = torch.zeros(30, dtype=torch.int32, device="cuda")
        p = _lib.IcpParams()
        call = lambda: ops.icp(sp, so1, tp, to1, g, len(src), len(tgt), p, src_id=ids, tgt_id=ids, ctx=ctx)
        t_call, out = events(call, a.reps)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        build = icp = 0.0
        for ev in prof.key_averages():
            us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            if "icp3_kernel" in ev.key or "icp3_map_kernel" in ev.key:
                icp += us
            elif any(k in ev.key for k in ("map_", "Radix", "Scan", "icp3_map_z")):
                build += us
        want = o3.icp3_many([(src, tgt, gg) for gg in guesses])
        icpo = pcl.ICP()
        icpo.params = _lib.IcpParams()
        icpo.compute_batch(src, tgt, guesses)
        t0 = time.perf_counter()
        for _ in range(a.reps):
            res = icpo.compute_batch(src, tgt, guesses)
        t_host = (time.perf_counter() - t0) / a.reps * 1e3
        t0 = time.perf_counter()
        o3.icp3(src, tgt, guesses[0])
        t_orc = (time.perf_counter() - t0) * 1e3
        rows.append(dict(row="closure", n_target=n_target, guesses=30, ms_call=t_call, ms_grid_build=build / 1e3,
                         ms_icp_kernel=icp / 1e3, ms_compute_batch=t_host, ms_oracle_one_guess_one_thread=t_orc,
                         exact=exact(out, want) and exact(res, want)))
    t0 = time.perf_counter()
    o3.icp3(srcs[0], tgts[0], None, orc.IcpParams(**FIXED20))
    rows.append(dict(row="oracle", problem="config3 fixed20", ms_one_thread=(time.perf_counter() - t0) * 1e3, exact=True))

    res = dict(card=card, rows=rows)
    for r in rows:
        print(json.dumps(r))
    print("card:", card)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    assert all(r["exact"] for r in rows), "a row differs from the oracle"


if __name__ == "__main__":
    main()
