"""Loop-closure covariance (row N1) timing: SLAM.compute_icp_with_cov_batch over a backlog of candidates -- one ICP
launch for every candidate's guesses, one MinCovDet launch -- end to end and by part, next to sklearn's MinCovDet fit
(what compute_icp_with_cov calls, slam.py:365-371) on a sample of the same candidates.  Prints one JSON line and writes
nothing.
Run on an H100:  PYTHONPATH=. python tools/bench_n1_icp_cov.py [--candidates N] [--device D]

Workload: N candidates (default 1024) built from 32 seeded synth.make_icp_pair scenes, source ~1 500 points (a
5-keyframe aggregate), target ~4 000, 30 guesses each drawn around the true pose with the spread of
tests/test_dropin_gpu.py::test_slam_scan_matching_surface (0.2 m, 0.2 m, 0.02 rad).

  candidates_per_s   N / end-to-end wall time (median of 3, after one warm-up call)
  ms_icp_launch      ICP.compute_pairs alone: the one sfe_icp_batch_host call, copies included
  ms_host_draws      the trial supports of every fitted candidate (30 permutations each from numpy's generator)
  ms_mcd_kernel      the MinCovDet kernel alone, CUDA events, inputs already on the device
  ms_mcd_host_call   sfe_mincovdet_host, copies included
  ms_host_rest       end to end minus ICP, draws and the MinCovDet call: sample forming, packing, local-frame
                     rotation, determinant test
  sklearn_*          sklearn's MinCovDet on 32 of the fitted candidates: ms per fit on this host, and how many of the 32
                     the device reproduces (status equal, location and covariance within rtol 1e-9, atol 1e-15)
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def run(N, device=0, n_scenes=32, reps=3):
    import torch
    from sklearn.covariance import MinCovDet

    from sonar_slam_b200 import _lib, mcd, ops, synth
    from sonar_slam_b200.bruce_slam.slam import SLAM, Pose2
    torch.cuda.set_device(device)
    rng = np.random.default_rng(0)
    scenes = [synth.make_icp_pair(1000 + k, n_source=1500, n_target=4000) for k in range(n_scenes)]
    problems = []
    for c in range(N):
        src, tgt, T = scenes[c % n_scenes]
        true = np.array([T[0, 2], T[1, 2], np.arctan2(T[1, 0], T[0, 0])])
        problems.append((src, tgt, [Pose2(*(true + rng.normal(0, [0.2, 0.2, 0.02]))) for _ in range(30)]))
    slam = SLAM()
    slam.icp.params = _lib.IcpParams()   # the shipped icp.yaml chain
    np.random.seed(0)
    slam.compute_icp_with_cov_batch(problems)                        # warm-up (allocations, library load)
    e2e = []
    for _ in range(reps):
        np.random.seed(0)
        t0 = time.perf_counter()
        out = slam.compute_icp_with_cov_batch(problems)
        e2e.append(time.perf_counter() - t0)
    e2e_s = float(np.median(e2e))
    # the parts, each alone on the same input
    t0 = time.perf_counter()
    res = slam.icp.compute_pairs([p[0] for p in problems], [p[1] for p in problems],
                                 [[g.matrix() for g in p[2]] for p in problems])
    icp_s = time.perf_counter() - t0
    samples = [np.array([(T[0, 2], T[1, 2], np.arctan2(T[1, 0], T[0, 0]))
                         for m, T in zip(r["messages"], r["T"]) if m == "success"]) for r in res]
    fit = [s for s in samples if len(s) >= mcd.MIN_SAMPLES]
    np.random.seed(0)
    t0 = time.perf_counter()
    subsets = np.stack([mcd.draw_trial_supports(len(s)) for s in fit])
    draws_s = time.perf_counter() - t0
    X, n = mcd.pack(fit)
    t0 = time.perf_counter()
    mcd.mincovdet_host(X, n, subsets, float32=True)
    mcd_call_s = time.perf_counter() - t0
    Xd, nd, Sd = (torch.from_numpy(a).to(f"cuda:{device}") for a in (X, n, subsets))
    ops.mincovdet(Xd, nd, Sd, float32=True)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    ops.mincovdet(Xd, nd, Sd, float32=True)
    b.record()
    torch.cuda.synchronize()
    kernel_ms = a.elapsed_time(b)
    # sklearn's fit on 32 candidates, from the supports the device gets
    k = min(32, len(fit))
    sk_s, agree = 0.0, 0
    sup = [mcd.draw_trial_supports(len(fit[i]), np.random.RandomState(i)) for i in range(k)]
    dev = mcd.mincovdet_host(X[:k], n[:k], np.stack(sup), float32=True)
    for i in range(k):
        t0 = time.perf_counter()
        try:
            f = MinCovDet(store_precision=False, support_fraction=0.8, random_state=np.random.RandomState(i)).fit(fit[i])
            want = (mcd.OK, f.location_, f.covariance_)
        except ValueError:
            want = (mcd.ZERO_COV, None, None)
        sk_s += time.perf_counter() - t0
        if dev["status"][i] == want[0] and (want[0] != mcd.OK or (
                np.allclose(dev["location"][i], want[1], rtol=1e-9, atol=1e-15)
                and np.allclose(dev["covariance"][i], want[2], rtol=1e-9, atol=1e-15))):
            agree += 1
    from bench import gpu_info   # card name and power limit, read only
    return {"metric": "loop-closure candidates/s (ICP x 30 + MinCovDet)", "gpu": gpu_info(device),
            "candidates": N, "guesses_per_candidate": 30, "source_points": 1500, "target_points": 4000,
            "distinct_scenes": n_scenes, "fits": len(fit), "successes": sum(o[0] == "success" for o in out),
            "candidates_per_s": N / e2e_s, "ms_end_to_end": e2e_s * 1e3,
            "ms_icp_launch": icp_s * 1e3, "ms_host_draws": draws_s * 1e3, "ms_mcd_kernel": kernel_ms,
            "ms_mcd_host_call": mcd_call_s * 1e3,
            "ms_host_rest": (e2e_s - icp_s - draws_s - mcd_call_s) * 1e3,
            "sklearn_ms_per_fit": sk_s / max(1, k) * 1e3, "sklearn_sample": k, "sklearn_agree": agree}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--candidates", type=int, default=1024)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    print(json.dumps(run(a.candidates, a.device)), flush=True)
