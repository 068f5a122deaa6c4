import numpy as np, torch
from sonar_slam_b200 import _lib, ops, synth
P = torch.cuda.get_device_properties(0).multi_processor_count  # one wave: one problem per SM
pairs = [synth.make_icp_pair(s)[:2] for s in range(4)]
def pack(ns=None, nt=None):
    src = np.concatenate([pairs[i % 4][0][:ns] for i in range(P)]); tgt = np.concatenate([pairs[i % 4][1][:nt] for i in range(P)])
    so = np.zeros(P + 1, np.int32); so[1:] = np.cumsum([len(pairs[i % 4][0][:ns]) for i in range(P)])
    to = np.zeros(P + 1, np.int32); to[1:] = np.cumsum([len(pairs[i % 4][1][:nt]) for i in range(P)])
    return torch.from_numpy(src).cuda(), torch.from_numpy(so).cuda(), torch.from_numpy(tgt).cuda(), torch.from_numpy(to).cuda()
gs = torch.eye(3, device="cuda").repeat(P, 1, 1).contiguous()
def t(args, prm, ns, nt):
    for _ in range(2): ops.icp(*args[:2], *args[2:], gs, ns, nt, prm)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); ops.icp(*args[:2], *args[2:], gs, ns, nt, prm); e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1)
a = pack()
for it in (1, 2, 5, 10, 20, 40):
    print("2k/20k iters", it, "ms", round(t(a, _lib.IcpParams(smooth_length=0, max_iterations=it), 2000, 20000), 3))
b = pack(2000, 5000)
for it in (1, 20):
    print("2k/5k iters", it, "ms", round(t(b, _lib.IcpParams(smooth_length=0, max_iterations=it), 2000, 5000), 3))
c = pack(500, 20000)
for it in (1, 20):
    print("500/20k iters", it, "ms", round(t(c, _lib.IcpParams(smooth_length=0, max_iterations=it), 500, 20000), 3))
