"""Multi-GPU batching of the front end: one process per GPU, frames sharded by rank.

The per-keyframe path is embarrassingly parallel given the odometry poses (SURVEY.md 8(e)); the only
coupling between neighbouring frames is the scan-matching window (frame i is matched against frames
i-window .. i-1), so every shard carries `window` halo frames in front of it whose clouds are recomputed
locally and whose results are dropped.  torch.distributed (NCCL on GPUs, gloo on CPU for tests) is used
only at the edges: scatter the backlog from rank 0 (send / recv), gather the per-frame results (one tensor gather
per result field).
"""
import numpy as np
import torch
import torch.distributed as dist


def shard_bounds(n, world):
    """Contiguous, near-equal blocks: list of (start, end) for every rank."""
    per, extra = divmod(n, world)
    out, s = [], 0
    for r in range(world):
        e = s + per + (1 if r < extra else 0)
        out.append((s, e))
        s = e
    return out


def shard_with_halo(n, world, window):
    """(halo_start, start, end) per rank: rank r processes frames [halo_start, end) and reports [start, end)."""
    return [(max(0, s - window), s, e) for s, e in shard_bounds(n, world)]


def scatter_backlog(frames, poses, window, device="cpu", src=0):
    """Rank `src` holds frames uint8 [n,R,B] and poses float64 [n,3] (others pass None); every rank
    returns (frames_local, poses_local, n_halo) as torch tensors on `device`."""
    rank, world = dist.get_rank(), dist.get_world_size()
    meta = [None]
    if rank == src:
        meta = [(tuple(frames.shape), window)]
    dist.broadcast_object_list(meta, src=src)
    (n, R, B), window = meta[0]
    plan = shard_with_halo(n, world, window)
    h, s, e = plan[rank]
    f_local = torch.empty((e - h, R, B), dtype=torch.uint8, device=device)
    p_local = torch.empty((e - h, 3), dtype=torch.float64, device=device)
    if rank == src:
        ft = torch.as_tensor(frames).to(device)
        pt = torch.as_tensor(poses, dtype=torch.float64).to(device)
        reqs = []
        for r, (hh, ss, ee) in enumerate(plan):
            if r == src:
                f_local.copy_(ft[hh:ee])
                p_local.copy_(pt[hh:ee])
            else:
                reqs.append(dist.isend(ft[hh:ee].contiguous(), dst=r))
                reqs.append(dist.isend(pt[hh:ee].contiguous(), dst=r))
        for q in reqs:
            q.wait()
    else:
        dist.recv(f_local, src=src)
        dist.recv(p_local, src=src)
    return f_local, p_local, s - h


def gather_results(local, n_halo, n_total, dst=0, device=None):
    """local: dict of per-frame numpy arrays for the rank's [halo_start, end) frames.  Rank `dst` gets the
    concatenation over ranks in frame order with halos removed (others get None).  The first frame of
    every shard but the first keeps its halo-informed result; frame 0 of the backlog stays "skipped".

    One `dist.gather` of a tensor per key (NCCL on GPUs, gloo in the CPU tests; no pickling): every rank knows every
    shard's length from `shard_bounds(n_total, world)`, shards are padded to the longest one for the collective."""
    rank, world = dist.get_rank(), dist.get_world_size()
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else "cpu"
    lens = [e - s for s, e in shard_bounds(n_total, world)]
    longest = max(lens) if lens else 0
    out = {}
    for k in sorted(local):
        own = torch.from_numpy(np.ascontiguousarray(local[k][n_halo:])).to(device)
        assert own.shape[0] == lens[rank], (k, own.shape, lens[rank])
        pad = torch.zeros((longest,) + tuple(own.shape[1:]), dtype=own.dtype, device=device)
        pad[:own.shape[0]] = own
        bufs = [torch.empty_like(pad) for _ in range(world)] if rank == dst else None
        dist.gather(pad, bufs, dst=dst)
        if rank == dst:
            out[k] = torch.cat([b[:n] for b, n in zip(bufs, lens)]).cpu().numpy()
    if rank != dst:
        return None
    assert all(len(v) == n_total for v in out.values())
    return out


# ------------------------------------------------------------------------------------------------------------------
# Backlog of independent scan matches (BASELINE config 5; SURVEY.md 8(e)): P (source, target, guess) problems held
# by rank `src` are sharded in contiguous blocks (shard_bounds), streamed to their ranks with grouped NCCL
# send/recv (dist.batch_isend_irecv = one ncclGroup per chunk), solved with the batched ICP kernel, and the
# 48-byte results are gathered back with NCCL.  Clouds of one backlog have a common size (ns / nt points: the
# benchmark's 2 k / 20 k; real clouds are padded by the caller), so a problem is a fixed-size record and no offsets
# travel.  No collective sits inside the algorithm: the scatter and the gather are the only communication.
RESULT_WORDS = 12  # T (9 float32) + iterations, inliers, status (int32) = 48 B per problem


def _rank_world():
    """(rank, world); (0, 1) when no process group was initialised (single-GPU use)."""
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def chunk_plan(P, world, chunks):
    """Every rank's shard is cut into the same number of chunks: plan[r] = [(start, end), ...] (global indices);
    a chunk may be empty.  Shared by sender and receivers so that their send/recv sizes agree."""
    plan = []
    for s, e in shard_bounds(P, world):
        n = e - s
        per = -(-n // chunks) if n else 0
        plan.append([(min(s + c * per, e), min(s + (c + 1) * per, e)) for c in range(chunks)])
    return plan


def pack_results(res):
    """dict(T [n,3,3] f32, iterations, inliers, status i32) -> int32 [n, RESULT_WORDS]."""
    n = res["T"].shape[0]
    out = torch.empty((n, RESULT_WORDS), dtype=torch.int32, device=res["T"].device)
    out[:, :9] = res["T"].reshape(n, 9).contiguous().view(torch.int32)
    out[:, 9], out[:, 10], out[:, 11] = res["iterations"], res["inliers"], res["status"]
    return out


def unpack_results(packed):
    return dict(T=packed[:, :9].contiguous().view(torch.float32).reshape(-1, 3, 3), iterations=packed[:, 9],
                inliers=packed[:, 10], status=packed[:, 11])


_STREAMS = {}


def _side_streams(dev):
    if dev not in _STREAMS:
        _STREAMS[dev] = (torch.cuda.Stream(dev), [torch.cuda.Stream(dev), torch.cuda.Stream(dev)])
    return _STREAMS[dev]


def _default_icp(src, tgt, guess, prm):
    """src [n, ns, 2], tgt [n, nt, 2], guess [n,3,3] cuda tensors -> packed results [n, RESULT_WORDS]."""
    from . import ops
    n, ns, nt = src.shape[0], src.shape[1], tgt.shape[1]
    dev = src.device
    so = torch.arange(n + 1, dtype=torch.int32, device=dev) * ns
    to = torch.arange(n + 1, dtype=torch.int32, device=dev) * nt
    return pack_results(ops.icp(src.reshape(-1, 2), so, tgt.reshape(-1, 2), to, guess, ns, nt, prm))


def scatter_pairs(P, ns, nt, src_all=None, tgt_all=None, guess_all=None, src=0, device="cuda"):
    """One grouped send/recv: rank `src` holds src_all [P,ns,2], tgt_all [P,nt,2], guess_all [P,3,3] (float32, on
    its device); every rank returns its shard (src, tgt, guess) -- views into the originals on rank `src`."""
    rank, world = _rank_world()
    s, e = shard_bounds(P, world)[rank]
    if rank == src:
        ops_ = []
        for r, (a, b) in enumerate(shard_bounds(P, world)):
            if r != src and b > a:
                ops_ += [dist.P2POp(dist.isend, src_all[a:b], r), dist.P2POp(dist.isend, tgt_all[a:b], r),
                         dist.P2POp(dist.isend, guess_all[a:b], r)]
        for q in (dist.batch_isend_irecv(ops_) if ops_ else []):
            q.wait()
        return src_all[s:e], tgt_all[s:e], guess_all[s:e]
    n = e - s
    out = (torch.empty((n, ns, 2), dtype=torch.float32, device=device),
           torch.empty((n, nt, 2), dtype=torch.float32, device=device),
           torch.empty((n, 3, 3), dtype=torch.float32, device=device))
    if n:
        for q in dist.batch_isend_irecv([dist.P2POp(dist.irecv, t, src) for t in out]):
            q.wait()
    return out


def gather_pair_results(local_packed, P, dst=0):
    """NCCL gather of the packed results (shards padded to the largest one); rank `dst` gets [P, RESULT_WORDS]."""
    rank, world = _rank_world()
    bounds = shard_bounds(P, world)
    if world == 1:
        return local_packed
    n_max = max(e - s for s, e in bounds)
    pad = torch.zeros((n_max, RESULT_WORDS), dtype=torch.int32, device=local_packed.device)
    pad[:local_packed.shape[0]] = local_packed
    parts = [torch.empty_like(pad) for _ in range(world)] if rank == dst else None
    dist.gather(pad, parts, dst=dst)
    if rank != dst:
        return None
    return torch.cat([parts[r][:e - s] for r, (s, e) in enumerate(bounds)])


def run_pair_backlog(P, ns, nt, prm, src_all=None, tgt_all=None, guess_all=None, chunks=8, src=0, icp_fn=None,
                     device="cuda"):
    """The whole config-5 step with the scatter hidden behind the solver: every shard is cut into `chunks` pieces,
    each sent as one NCCL group on a communication stream; a rank starts solving piece c as soon as it has arrived
    while the later pieces are still in flight; rank `src` solves its own shard straight from the backlog.  Returns the packed results [P, RESULT_WORDS] on rank `src`
    (None elsewhere).  `icp_fn(src, tgt, guess, prm) -> packed` is injectable (CPU tests run this over gloo)."""
    icp_fn = icp_fn or _default_icp
    rank, world = _rank_world()
    plan = chunk_plan(P, world, chunks)
    s, e = shard_bounds(P, world)[rank]
    cuda = torch.device(device).type == "cuda"
    local = torch.empty((e - s, RESULT_WORDS), dtype=torch.int32, device=device)
    if world == 1:
        for a, b in plan[0]:
            if b > a:
                local[a - s:b - s] = icp_fn(src_all[a:b], tgt_all[a:b], guess_all[a:b], prm)
        return local
    compute = torch.cuda.current_stream() if cuda else None
    # the pieces are solved on two alternating streams: a piece is one launch of one CTA per problem, and its last,
    # partly filled wave of CTAs would otherwise idle most SMs once per piece.
    # (the side streams are created once per device and reused: libsonarfe contexts are cached per stream)
    comm, solve = _side_streams(torch.cuda.current_device()) if cuda else (None, [None, None])
    if cuda:
        comm.wait_stream(compute)
        for st in solve:
            st.wait_stream(compute)

    def on_comm():
        return torch.cuda.stream(comm) if cuda else _Null()

    def on_solve(c):
        return torch.cuda.stream(solve[c & 1]) if cuda else _Null()

    if rank == src:
        # stream every other rank's pieces out, chunk by chunk (one NCCL group per chunk), while solving our own
        for c in range(chunks):
            ops_ = []
            for r in range(world):
                a, b = plan[r][c]
                if r != src and b > a:
                    ops_ += [dist.P2POp(dist.isend, src_all[a:b], r), dist.P2POp(dist.isend, tgt_all[a:b], r),
                             dist.P2POp(dist.isend, guess_all[a:b], r)]
            with on_comm():
                for q in (dist.batch_isend_irecv(ops_) if ops_ else []):
                    q.wait()
            a, b = plan[src][c]
            if b > a:
                with on_solve(c):
                    local[a - s:b - s] = icp_fn(src_all[a:b], tgt_all[a:b], guess_all[a:b], prm)
    else:
        # The whole shard is received into its final place (memory is not the constraint: 176 KB per pair), every
        # piece as its own grouped recv posted up front on the communication stream: the sender never waits for a
        # buffer to free up -- a send kernel parked on the sender's SMs until the receiver's solver drains slows
        # the sender down -- and the solver starts on piece c as soon as piece c is there.
        n_loc = e - s
        sb = torch.empty((n_loc, ns, 2), dtype=torch.float32, device=device)
        tb = torch.empty((n_loc, nt, 2), dtype=torch.float32, device=device)
        gb = torch.empty((n_loc, 3, 3), dtype=torch.float32, device=device)
        ready = [torch.cuda.Event() for _ in range(chunks)] if cuda else None
        with on_comm():
            for c in range(chunks):
                a, b = plan[rank][c]
                if b <= a:
                    continue
                for q in dist.batch_isend_irecv([dist.P2POp(dist.irecv, t[a - s:b - s], src) for t in (sb, tb, gb)]):
                    q.wait()
                if cuda:
                    ready[c].record(comm)
        for c in range(chunks):
            a, b = plan[rank][c]
            if b <= a:
                continue
            with on_solve(c):
                if cuda:
                    solve[c & 1].wait_event(ready[c])
                local[a - s:b - s] = icp_fn(sb[a - s:b - s], tb[a - s:b - s], gb[a - s:b - s], prm)
    if cuda:
        for st in solve:
            compute.wait_stream(st)
    if cuda:
        compute.wait_stream(comm)
    return gather_pair_results(local, P, dst=src)


class _Null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False
