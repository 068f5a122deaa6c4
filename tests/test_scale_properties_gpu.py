"""GPU, BASELINE-sized inputs: size-independent properties instead of a CPU oracle pass over everything
(the oracle would need minutes per configuration); a random sample is still checked against the oracle."""
import numpy as np
import pytest
import torch

from oracle import featx_ref, oracle as orc, pipeline_ref
from sonar_slam_b200 import _lib, ops, pipeline, synth

pytestmark = pytest.mark.gpu
TAU = 2.749063720096473


def _rayleigh_frames(F, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((F, 512, 512), dtype=torch.uint8, device="cuda")
    for i in range(0, F, 512):
        n = min(512, F - i)
        u = torch.rand((n, 512, 512), device="cuda", generator=g).clamp_min(1e-7)
        out[i:i + n] = torch.clamp(torch.round(18.0 * torch.sqrt(-2.0 * torch.log(u))), 0, 255).to(torch.uint8)
    return out


def test_config2_4096_frames_cfar(gpu_ctx):
    """4096 x 512 x 512: u8 and f32 storage agree, bit plane == byte mask, borders empty, batch position
    irrelevant, and a sample of frames equals the oracle bit for bit."""
    F = 4096
    imgs = _rayleigh_frames(F, 7)
    a = ops.cfar(imgs, "SOCA", 20, 5, TAU, gate=65, want_bits=True)
    mask, bits = a["mask"], a["bits"]
    w = bits.view(torch.int32)
    unpacked = ((w.unsqueeze(-1) >> torch.arange(32, device="cuda", dtype=torch.int32)) & 1).to(torch.uint8).reshape(F, 512, 512)
    assert torch.equal(unpacked, mask)
    del unpacked
    assert int(mask[:, :25].sum()) == 0 and int(mask[:, -25:].sum()) == 0
    for lo in range(0, F, 1024):            # f32 copy in slices (4 GiB as float32 otherwise)
        b = ops.cfar(imgs[lo:lo + 1024].float(), "SOCA", 20, 5, TAU, gate=65)["mask"]
        assert torch.equal(b, mask[lo:lo + 1024])
    perm = torch.randperm(F, device="cuda")[:512]
    c = ops.cfar(imgs[perm].contiguous(), "SOCA", 20, 5, TAU, gate=65)["mask"]
    assert torch.equal(c, mask[perm])
    for f in (0, 1234, 4095):
        want = orc.cfar_u8("SOCA", imgs[f].cpu().numpy(), 20, 5, 0, TAU, 65)
        assert np.array_equal(mask[f].cpu().numpy(), want)


def test_config5_style_icp_batch_is_order_independent(gpu_ctx):
    """2048 config-3 sized pairs (8 distinct, repeated): every copy of a pair gives the identical result
    wherever it sits in the batch; a sample equals the oracle within the north-star tolerances."""
    base = [synth.make_icp_pair(s)[:2] for s in range(8)]
    P = 2048
    rng = np.random.default_rng(0)
    which = rng.integers(0, 8, P)
    src = np.concatenate([base[k][0] for k in which])
    tgt = np.concatenate([base[k][1] for k in which])
    so = np.zeros(P + 1, np.int32)
    so[1:] = np.cumsum([len(base[k][0]) for k in which])
    to = np.zeros(P + 1, np.int32)
    to[1:] = np.cumsum([len(base[k][1]) for k in which])
    prm = _lib.IcpParams(smooth_length=0, max_iterations=20)
    out = ops.icp(torch.from_numpy(src).cuda(), torch.from_numpy(so).cuda(), torch.from_numpy(tgt).cuda(),
                  torch.from_numpy(to).cuda(), torch.eye(3, device="cuda").repeat(P, 1, 1).contiguous(), 2000, 20000, prm)
    T = out["T"].cpu().numpy()
    inl = out["inliers"].cpu().numpy()
    assert (out["status"].cpu().numpy() == 0).all() and (out["iterations"].cpu().numpy() == 20).all()
    for k in range(8):
        sel = np.nonzero(which == k)[0]
        assert np.array_equal(T[sel], np.repeat(T[sel[:1]], len(sel), 0)) and len(set(inl[sel].tolist())) == 1
        want = orc.icp(base[k][0], base[k][1], None, orc.IcpParams(smooth_length=0, max_iterations=20))
        assert inl[sel[0]] == want["inliers"]
        assert np.array_equal(T[sel[0]].view(np.uint32), want["T"].view(np.uint32))   # default mode: the oracle's bits
    # the same backlog through the config-5 entry point (one rank: no scatter, pieces of the shard one after the other)
    from sonar_slam_b200 import dist as sdist
    fixed = [k for k in range(8) if len(base[k][1]) == 20000]
    if fixed:
        pick = np.array([fixed[i % len(fixed)] for i in range(300)])
        S = torch.from_numpy(np.stack([base[k][0] for k in pick])).cuda()
        Tg = torch.from_numpy(np.stack([base[k][1] for k in pick])).cuda()
        G = torch.eye(3, device="cuda").repeat(len(pick), 1, 1).contiguous()
        packed = sdist.run_pair_backlog(len(pick), 2000, 20000, prm, S, Tg, G, chunks=4)
        res = sdist.unpack_results(packed)
        for j, k in enumerate(pick):
            first = np.nonzero(which == k)[0][0]
            assert np.array_equal(res["T"][j].cpu().numpy().view(np.uint32), T[first].view(np.uint32))
            assert int(res["inliers"][j]) == inl[first] and int(res["status"][j]) == 0


def test_config4_replay_chunking_and_batch_alignment(gpu_ctx):
    """1024-frame replay: the host call (any chunk size) equals the device-resident call, a sub-range replayed
    on its own gives the same edges once its window is warm, and sampled frames equal the oracle chain."""
    n = 1024
    d = synth.make_trajectory_frames(n, seed=5, device="cuda")
    frames_dev, poses = d["frames"], d["poses_odom"]
    frames = frames_dev.cpu().numpy()
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(gpu_ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    fe = pipeline.FrontEnd(gpu_ctx, maps, max_frames=n, tau=TAU)
    a = fe.run_host(frames, poses, chunk_frames=100)
    b = fe.run_host(frames, poses, chunk_frames=1024)
    fe.run_dev(frames_dev.data_ptr(), poses, n)
    r = fe.results_dev()
    Td = gpu_ctx.to_host(r["T"], (n, 3, 3), np.float32)
    for k in ("T", "status", "iterations", "inliers", "npoints"):
        assert np.array_equal(a[k], b[k]), k
    assert np.array_equal(a["T"], Td)
    lo, hi = 300, 400
    sub = fe.run_host(frames[lo:hi], poses[lo:hi], chunk_frames=64)
    assert np.array_equal(sub["T"][3:], a["T"][lo + 3:hi]) and np.array_equal(sub["npoints"], a["npoints"][lo:hi])
    assert (a["status"][1:] == 0).mean() > 0.9
    # oracle on a window of frames
    s0 = 500
    clouds, want = pipeline_ref.run(frames[s0:s0 + 8], poses[s0:s0 + 8], geo, icp_params=orc.IcpParams())
    for i in range(3, 8):   # the default ICP mode is the oracle's float32 chain: bit for bit (DESIGN.md section 2)
        assert a["npoints"][s0 + i] == len(clouds[i]) and a["status"][s0 + i] == want[i]["status"]
        if want[i]["status"] == 0:
            assert a["inliers"][s0 + i] == want[i]["inliers"] and a["iterations"][s0 + i] == want[i]["iterations"]
        assert np.array_equal(a["T"][s0 + i].view(np.uint32), np.asarray(want[i]["T"], np.float32).view(np.uint32)), \
            (s0 + i, a["T"][s0 + i], want[i]["T"])
