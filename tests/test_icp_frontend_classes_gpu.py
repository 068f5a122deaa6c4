"""GPU: the batched front end's ICP size classes (pipeline.cu: FE_ICP_CLASSES, icp.cu: icp_run's class path) equal
the oracle (oracle/icp_ref.c) bit for bit -- status, iterations, inliers and every bit of T -- on problems on both
sides of the class bound, in batches that fill every class, leave one empty, or are smaller than one wave; and
every problem is in exactly one class's work list, the class it fits first, at a place that follows the largest-first
order (source size in 32-point steps, ties by index)."""
import ctypes

import numpy as np
import pytest

from oracle import oracle as orc
from sonar_slam_b200 import synth

pytestmark = pytest.mark.gpu

F32 = np.float32
SMALL = (640, 800)    # pipeline.cu: FE_ICP_SMALL_SRC / _TGT (128-thread CTAs); then the capacity class
SETTINGS = {"point": {}, "plane": dict(minimizer=1, normals_knn=5)}


def _pair(ns, nt, seed):
    """synth.make_icp_pair with exactly ns / nt points (target topped up with jittered wall points)."""
    s, t, T = synth.make_icp_pair(seed, n_source=ns, n_target=nt)
    if len(t) < nt:
        rng = np.random.default_rng(seed)
        extra = t[rng.integers(len(t), size=nt - len(t))] + rng.normal(0, 0.03, (nt - len(t), 2))
        t = np.concatenate([t, extra]).astype(F32)
    assert (len(s), len(t)) == (ns, nt)
    rng = np.random.default_rng(seed + 1)
    guess = (np.asarray(T, np.float64) @ synth.se2(*rng.normal(0, (0.2, 0.2, 0.02)))).astype(F32)
    return s, t, guess


def expected_class(ns, nt):
    return 0 if ns <= SMALL[0] and nt <= SMALL[1] else 1


def run(sizes, setting, seed=0):
    import torch
    from sonar_slam_b200 import _lib, ops
    probs = [_pair(ns, nt, seed + 7 * k) for k, (ns, nt) in enumerate(sizes)]
    P = len(probs)
    dev = "cuda:0"
    src = torch.from_numpy(np.concatenate([p[0] for p in probs])).to(dev)
    tgt = torch.from_numpy(np.concatenate([p[1] for p in probs])).to(dev)
    soff = torch.tensor(np.cumsum([0] + [len(p[0]) for p in probs]), dtype=torch.int32, device=dev)
    toff = torch.tensor(np.cumsum([0] + [len(p[1]) for p in probs]), dtype=torch.int32, device=dev)
    guess = torch.from_numpy(np.stack([p[2] for p in probs])).to(dev)
    T = torch.empty((P, 3, 3), dtype=torch.float32, device=dev)
    iters, inl, st = (torch.empty(P, dtype=torch.int32, device=dev) for _ in range(3))
    cls = torch.full((2 * P,), -1, dtype=torch.int32, device=dev)
    ctx = ops.context(0)
    prm = _lib.IcpParams(**SETTINGS[setting])
    p_ = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    _lib.check(ctx.lib.sfe_frontend_icp_dev(ctx.handle, ctypes.byref(prm), p_(src), p_(soff), p_(tgt), p_(toff), P,
                                            max(s for s, _ in sizes), max(t for _, t in sizes), p_(guess), p_(T),
                                            p_(iters), p_(inl), p_(st), p_(cls)), "sfe_frontend_icp_dev")
    torch.cuda.synchronize()
    res = dict(T=T.cpu().numpy(), iterations=iters.cpu().numpy(), inliers=inl.cpu().numpy(), status=st.cpu().numpy())
    cls = cls.cpu().numpy()

    # every problem in exactly one list, in the class it fits first, at its largest-first place
    klass, place = cls[:P], cls[P:]
    assert klass.tolist() == [expected_class(*s) for s in sizes], klass
    for c in range(2):
        members = np.flatnonzero(klass == c)
        assert sorted(place[members].tolist()) == list(range(len(members))), (c, place[members])
        order = members[np.argsort(place[members])]
        key = [(-min(sizes[p][0] // 32, 31), p) for p in order]
        assert key == sorted(key), (c, order)

    oprm = orc.IcpParams(**SETTINGS[setting])
    for k, (s, t, g) in enumerate(probs):
        want = orc.icp(s, t, g, oprm)
        got = (int(res["status"][k]), int(res["iterations"][k]), int(res["inliers"][k]))
        assert got == (want["status"], want["iterations"], want["inliers"]), (setting, sizes[k], got, want)
        assert np.array_equal(res["T"][k].astype(F32).view(np.uint32), want["T"].view(np.uint32)), \
            (setting, sizes[k], res["T"][k], want["T"])


BOUNDS = [(SMALL[0], SMALL[1]), (SMALL[0] + 1, SMALL[1]), (SMALL[0], SMALL[1] + 1), (120, 200), (500, 300),
          (700, 1100)]


@pytest.mark.parametrize("setting", sorted(SETTINGS))
def test_class_bounds_on_both_axes_every_class_populated(setting):
    # the bound and bound + 1 on both axes; both classes (capacity included) hold problems
    run(BOUNDS, setting)


@pytest.mark.parametrize("setting", sorted(SETTINGS))
@pytest.mark.parametrize("sizes", [[(300, 400), (64, 100), (640, 800), (512, 700)], [(700, 500), (650, 1000), (641, 300)]],
                         ids=["capacity-empty", "small-empty"])
def test_one_class_empty(setting, sizes):
    run(sizes, setting, seed=11)


@pytest.mark.parametrize("setting", sorted(SETTINGS))
@pytest.mark.parametrize("sizes", [[(300, 420)], [(900, 1200)]], ids=["small", "capacity"])
def test_batch_of_one(setting, sizes):
    run(sizes, setting, seed=23)


@pytest.mark.parametrize("setting", sorted(SETTINGS))
def test_mixed_batch_fewer_than_one_wave(setting):
    # problems of mixed sizes in both classes, each class's list in largest-first order
    rng = np.random.default_rng(5)
    sizes = [(int(rng.integers(40, 700)), int(rng.integers(60, 950))) for _ in range(96)]
    run(sizes, setting, seed=31)
