"""ICP launch for ncu: config-3 pairs (2k source vs 20k target), fixed 20 iterations."""
import sys
import numpy as np, torch
from sonar_slam_b200 import _lib, ops, synth
P = int(sys.argv[1]) if len(sys.argv) > 1 else torch.cuda.get_device_properties(0).multi_processor_count
pairs = [synth.make_icp_pair(s)[:2] for s in range(4)]
src = np.concatenate([pairs[i % 4][0] for i in range(P)]); tgt = np.concatenate([pairs[i % 4][1] for i in range(P)])
so = np.zeros(P + 1, np.int32); so[1:] = np.cumsum([len(pairs[i % 4][0]) for i in range(P)])
to = np.zeros(P + 1, np.int32); to[1:] = np.cumsum([len(pairs[i % 4][1]) for i in range(P)])
sp, tp = torch.from_numpy(src).cuda(), torch.from_numpy(tgt).cuda()
so, to = torch.from_numpy(so).cuda(), torch.from_numpy(to).cuda()
gs = torch.eye(3, device="cuda").repeat(P, 1, 1).contiguous()
prm = _lib.IcpParams(smooth_length=0, max_iterations=20)
for _ in range(2):
    out = ops.icp(sp, so, tp, to, gs, 2000, 20000, prm)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); out = ops.icp(sp, so, tp, to, gs, 2000, 20000, prm); e1.record(); torch.cuda.synchronize()
print("ms", e0.elapsed_time(e1), "pairs", P, "inliers", out["inliers"][:4].tolist())
