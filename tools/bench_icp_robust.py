"""What a RobustOutlierFilter in the ICP chain (sfe_icp_set_robust) costs on the device, against the same call without
one, on the workloads of tools/bench_icp_voxel_filter.py.

Workloads:
  wave      the config-3 wave (132-SM-sized batches of 2 000-point sources on 20 000-point targets, 8 waves per call)
  frontend  the batched front end's ICP stage (sfe_frontend_icp_dev) on the frame clouds and window submaps of a
            512-frame bag
each without a robust filter and with every robustFct (tunings of tests/test_icp_robust_gpu.py), shipped checkers
(icp.yaml: MaxDist 3 m and Trimmed 0.8 stay on).  Per row:
  device_ms  the call on device tensors between two CUDA events, median of 5 after a warm-up call (wave: ms per wave)
  exact      the first three device results equal oracle/robust_ref.c's bit for bit (status, iterations, inliers, T)
Prints one JSON line with the card's name, power limit and SM clock, read in the same run.

    python tools/bench_icp_robust.py [--out FILE] [--only wave]
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
TUNING = {"cauchy": 0.05, "welsch": 0.1, "sc": 0.01, "gm": 0.02, "tukey": 0.2, "huber": 0.05, "L1": 1.0}


def measure(name, srcs, tgts, guesses, ids, fct, waves=1, frontend=False):
    """One call over P = len(guesses) problems, problem p: srcs[ids[p]] onto tgts[ids[p]] (ops.icp), or (srcs[p],
    tgts[p]) through sfe_frontend_icp_dev with the robust filter set on the context.  fct None: no robust filter."""
    import torch

    from oracle import oracle as orc
    from oracle import robust_ref as rr
    from sonar_slam_b200 import _lib, ops

    def pack(cl):
        off = np.zeros(len(cl) + 1, np.int32)
        off[1:] = np.cumsum([len(c) for c in cl])
        return torch.from_numpy(np.concatenate(cl).astype(F32)).cuda(), torch.from_numpy(off).cuda()

    sp, so = pack(srcs)
    tp, to = pack(tgts)
    si = torch.tensor(ids, dtype=torch.int32).cuda()
    g = torch.from_numpy(np.stack(guesses).astype(F32)).cuda()
    prm = _lib.IcpParams()
    rob = _lib.IcpRobust(fct, TUNING[fct]) if fct else None
    ctx = ops.context(0)
    if frontend:
        P = len(guesses)
        T = torch.empty((P, 3, 3), dtype=torch.float32, device="cuda")
        iters, inl, st = (torch.empty(P, dtype=torch.int32, device="cuda") for _ in range(3))
        p_ = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731

        def call():
            _lib.set_icp_robust(ctx, rob)
            _lib.check(ctx.lib.sfe_frontend_icp_dev(ctx.handle, ctypes.byref(prm), p_(sp), p_(so), p_(tp), p_(to), P,
                                                    max(map(len, srcs)), max(map(len, tgts)), p_(g), p_(T),
                                                    p_(iters), p_(inl), p_(st), None), "sfe_frontend_icp_dev")
            return dict(T=T, iterations=iters, inliers=inl, status=st)
    else:
        call = lambda: ops.icp(sp, so, tp, to, g, max(map(len, srcs)), max(map(len, tgts)), prm, src_id=si,  # noqa
                               tgt_id=si, robust=rob)
    res = call()
    torch.cuda.synchronize()
    dev = {k: v.cpu().numpy() for k, v in res.items()}
    orob = rr.Robust(fct, TUNING[fct]) if fct else None
    exact = True
    for k in range(min(3, len(guesses))):
        w = rr.icp(srcs[ids[k]], tgts[ids[k]], guesses[k], orc.IcpParams(), robust=orob)
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
    _lib.set_icp_robust(ctx, None)
    return dict(name=name, robust=fct, tuning=TUNING.get(fct), problems=len(guesses),
                status=[int(v) for v in dev["status"][:3]], iterations=[int(v) for v in dev["iterations"][:3]],
                device_ms=round(float(np.median(ev)) / waves, 3), exact=bool(exact))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", default=None, help="wave or frontend")
    args = ap.parse_args()
    import torch
    from bench_icp_voxel_filter import card, frontend_problems

    from sonar_slam_b200 import synth
    rows = []
    fcts = [None] + list(TUNING)
    if args.only in (None, "wave"):
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        waves = 8
        P = sms * waves
        pairs = [synth.make_icp_pair(1000 + k, n_source=2000, n_target=20000) for k in range(16)]
        ids = [k % 16 for k in range(P)]
        gs = [pairs[i][2].astype(F32) for i in ids]
        for fct in fcts:
            rows.append(measure("wave", [p[0] for p in pairs], [p[1] for p in pairs], gs, ids, fct, waves=waves))
            print(json.dumps(rows[-1]), file=sys.stderr)
    if args.only in (None, "frontend"):
        srcs, tgts, gs = frontend_problems(512)
        ids = list(range(len(gs)))
        for fct in fcts:
            rows.append(measure("frontend", srcs, tgts, gs, ids, fct, frontend=True))
            print(json.dumps(rows[-1]), file=sys.stderr)
    name, power, clock = card()
    line = json.dumps(dict(gpu=name, power_limit=power, sm_clock_max=clock, checkers="shipped", rows=rows))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
