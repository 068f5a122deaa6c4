"""Where the point-to-plane mode spends its time: ms per launch by iteration count, both minimisers, for the
config-3 size (one problem per SM: one wave) and the front end's size (4096 problems of ~360 x ~1000 points)."""
import numpy as np, torch
from sonar_slam_b200 import _lib, ops, synth


def pack(pairs, P):
    src = np.concatenate([pairs[i % len(pairs)][0] for i in range(P)]); tgt = np.concatenate([pairs[i % len(pairs)][1] for i in range(P)])
    so = np.zeros(P + 1, np.int32); so[1:] = np.cumsum([len(pairs[i % len(pairs)][0]) for i in range(P)])
    to = np.zeros(P + 1, np.int32); to[1:] = np.cumsum([len(pairs[i % len(pairs)][1]) for i in range(P)])
    return [torch.from_numpy(x).cuda() for x in (src, so, tgt, to)]


def t(a, g, prm, ns, nt):
    for _ in range(2): ops.icp(*a, g, ns, nt, prm)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); ops.icp(*a, g, ns, nt, prm); e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1)


big = [synth.make_icp_pair(s)[:2] for s in range(4)]
rng = np.random.default_rng(0)
small, gsm = [], []
for s in range(64):
    a, b, T = synth.make_icp_pair(5000 + s, n_source=int(rng.integers(300, 420)), n_target=int(rng.integers(900, 1100)))
    small.append((a, b)); gsm.append(T @ synth.se2(*rng.normal(0, [0.1, 0.1, 0.01])))
SMS = torch.cuda.get_device_properties(0).multi_processor_count
for name, pairs, P, ns, nt, g in ((f"2k/20k x{SMS}", big, SMS, 2000, 20000, None), ("360/1000 x4096", small, 4096, 640, 1100, gsm)):
    a = pack(pairs, P)
    gs = torch.eye(3, device="cuda").repeat(P, 1, 1).contiguous() if g is None else \
        torch.from_numpy(np.stack([g[i % len(g)] for i in range(P)]).astype(np.float32)).cuda()
    for mini, fl in ((0, 0), (1, 0)):
        print(name, "minimizer", mini, fl, {it: round(t(a, gs, _lib.IcpParams(smooth_length=0, max_iterations=it, minimizer=mini, flags=fl), ns, nt), 3)
                                        for it in (1, 2, 5, 10, 20)})
