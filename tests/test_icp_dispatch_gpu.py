"""GPU: the scan matcher equals the oracle (oracle/icp_ref.c) bit for bit -- status, iterations, inliers and every bit
of T -- in every launch class and search path `icp_run` can pick, and under every ICP setting `parse_icp_yaml`
accepts.

`dispatch` below restates the choice (icp.cu: icp_threads, icp_cta_smem, icp_kernel_for, icp_launch; the one-pass
test of icp_kernel_body.cuh) from the problem sizes and the device's limits, and every case asserts the class and path
it is meant to reach: 128 / 256 / 512-thread CTAs, <512, 2> and <512, 1>, the spatial source order, the trimmed cell
table at the in-CTA limit, one CTA per problem with the workspace slot taken from the SM id, the one-pass certified
search and the pruned three-pass search."""
import itertools

import numpy as np
import pytest

from oracle import oracle as orc
from sonar_slam_b200 import synth

pytestmark = pytest.mark.gpu

F32 = np.float32
FIXED20 = dict(max_iterations=20, smooth_length=0)
CHECKERS = {"fixed20": FIXED20, "shipped": {}}
FIELDS = ("matcher_max_dist", "outlier_max_dist", "trim_ratio", "max_iterations", "min_diff_rot", "min_diff_trans",
          "smooth_length", "flags", "minimizer", "normals_knn")

# ------------------------------------------------------------------ the dispatch table, restated
SHARED = 5712           # sizeof(IcpShared), rounded up to 16
RESERVED = 1024         # shared memory the driver reserves per CTA (sm_90)
GRID_MAX_CELLS = 16384
COARSE_WORDS = 96       # ICP_COARSE_WORDS: the coarse map is skipped above 96 * 32 coarse cells


def _dev():
    import torch
    p = torch.cuda.get_device_properties(0)
    return p.shared_memory_per_block_optin, p.shared_memory_per_multiprocessor, p.multi_processor_count


def icp_threads(ns_max):
    return 128 if ns_max <= 640 else (256 if ns_max <= 1536 else 512)


def layout(ns, nt, plane=False):
    """icp_cta_smem: (bytes, cell-table entries, trimmed) for an ns x nt layout."""
    optin = _dev()[0]
    order = ns > 1024

    def smem(mc):
        return (SHARED + 8 * nt + 4 * ((mc + 2) // 2 + 1) + 8 + 8 * ns + 4 * ns + 4 * ns + ns + 4 + 4 * ns
                + (2 * ns if order else 0) + 16 + (16 + 640 * 4 if plane and ns < 640 else 0))

    mc0 = mc = min(max(nt + nt // 2, 256), GRID_MAX_CELLS)
    while smem(mc) > optin and mc > nt // 4 + 256:
        mc -= mc // 8
    return smem(mc), mc, mc != mc0


def cta_limit(ns, plane=False):
    """Largest target icp_kernel lays out next to ns-point sources (above it: the map class)."""
    optin = _dev()[0]
    lo, hi = 0, 65535
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if layout(ns, mid, plane)[0] <= optin else (lo, mid - 1)
    return lo


def largest_source(nt):
    """Largest source the layout admits next to an nt-point target."""
    optin = _dev()[0]
    lo, hi = 1, 65535
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if layout(mid, nt)[0] <= optin else (lo, mid - 1)
    return lo


def dispatch(ns_max, nt_max, P, plane=False):
    """The launch class of one call: thread count, __launch_bounds__ minimum blocks, source order, CTAs per SM,
    workspace slot by SM id, trimmed cell table; 'map' when the targets exceed the in-CTA limit."""
    ns, nt = max(ns_max, 1), max(nt_max, 1)
    if nt > cta_limit(ns, plane):
        return dict(cls="map", threads=icp_threads(ns))
    _, sm_smem, sms = _dev()
    threads = icp_threads(ns)
    smem, _, trimmed = layout(ns, nt, plane)
    minb = {128: 7, 256: 4}.get(threads, 2 if smem <= 110 * 1024 else 1)
    per_sm = max(1, min(minb, sm_smem // (smem + RESERVED)))  # register-bound at MINB: the kernels sit at their cap
    return dict(cls=f"<{threads},{minb}>", threads=threads, minb=minb, order=ns > 1024, per_sm=per_sm,
                smid=per_sm == 1 and P > sms * per_sm, trimmed=trimmed)


def one_pass(ns, nt, threads):
    """icp_kernel_body.cuh: few, cheap searches take the one-pass certified path, the others the pruned passes."""
    return ns <= 5 * threads and nt <= 4096


def coarse_cells(tgt, max_cells):
    """cnx * cny of the pruned path's coarse occupancy map (grid.cuh grid_geometry on the centred target, float32)."""
    t = np.asarray(tgt, F32)
    m = np.cumsum(t, axis=0, dtype=F32)[-1] / F32(len(t))
    c = t - m
    w, h = c[:, 0].max() - c[:, 0].min(), c[:, 1].max() - c[:, 1].min()
    cell = F32(np.sqrt(F32(w * h) / F32(len(t))))
    cell = cell if cell > F32(0.05) else F32(0.05)
    for _ in range(32):
        inv = F32(1) / cell
        nx, ny = int(w * inv) + 1, int(h * inv) + 1
        if nx * ny <= max_cells and nx < 32768 and ny < 32768:
            break
        cell = cell * F32(1.5)
    inv = F32(1) / cell
    nx, ny = int(w * inv) + 1, int(h * inv) + 1
    return ((nx + 7) // 8) * ((ny + 7) // 8)


# ------------------------------------------------------------------ running and comparing
def _params(**kw):
    from sonar_slam_b200 import _lib
    return _lib.IcpParams(**kw), orc.IcpParams(**kw)


def _oracle_params(prm):
    return orc.IcpParams(**{f: getattr(prm, f) for f in FIELDS})


def _icp(prm):
    from sonar_slam_b200.bruce_slam import pcl
    icp = pcl.ICP()
    icp.params = prm
    return icp


def _guesses(T, k, seed, sd=(0.2, 0.2, 0.02)):
    rng = np.random.default_rng(seed)
    return [(np.asarray(T, np.float64) @ synth.se2(*rng.normal(0, sd))).astype(F32) for _ in range(k)]


def _pair(ns, nt, seed):
    """synth.make_icp_pair, its target topped up to exactly nt points (wall points jittered by 3 cm) when the thinned
    walls hold fewer."""
    s, t, T = synth.make_icp_pair(seed, n_source=ns, n_target=nt)
    if len(t) < nt:
        rng = np.random.default_rng(seed)
        extra = t[rng.integers(len(t), size=nt - len(t))] + rng.normal(0, 0.03, (nt - len(t), 2))
        t = np.concatenate([t, extra]).astype(F32)
    assert (len(s), len(t)) == (ns, nt), (len(s), len(t), ns, nt)
    return s, t, T


def _assert_equal(res, k, src, tgt, guess, oprm, tag=""):
    want = orc.icp(src, tgt, guess, oprm)
    got = (int(res["status"][k]), int(res["iterations"][k]), int(res["inliers"][k]))
    assert got == (want["status"], want["iterations"], want["inliers"]), (tag, k, got, want)
    assert np.array_equal(np.asarray(res["T"][k], F32).view(np.uint32), want["T"].view(np.uint32)), \
        (tag, k, res["T"][k], want["T"])
    return want


def run_pairs(pairs, prm):
    """pairs: [(src, tgt, [guesses])] in one compute_pairs call -> list of result dicts."""
    return _icp(prm).compute_pairs([p[0] for p in pairs], [p[1] for p in pairs], [p[2] for p in pairs])


def check_pairs(pairs, prm, oprm, tag=""):
    out = run_pairs(pairs, prm)
    wants = []
    for (s, t, gs), r in zip(pairs, out):
        wants.append([_assert_equal(r, k, s, t, g, oprm, tag) for k, g in enumerate(gs)])
    return out, wants


# ------------------------------------------------------------------ size grid: every class x path and boundary
def _size_calls():
    """(name, [(ns, nt)], guesses per pair, expected class, expected paths) -- one call each."""
    lim640, lim1536 = cta_limit(640), cta_limit(1536)
    big = largest_source(1000)
    return [
        ("128_onepass", [(1, 1), (2, 2), (639, 4095), (640, 4096), (640, 1), (1, 4096)], 2, "<128,7>", {True}),
        ("128_both", [(400, 4097), (640, 6000), (639, 4096), (2, 4097)], 2, "<128,7>", {True, False}),
        ("128_limit", [(400, lim640), (640, 12000), (640, 4097)], 2, "<128,7>", {False}),
        ("256_onepass", [(641, 1), (1024, 4096), (1000, 4095), (700, 2)], 2, "<256,4>", {True}),
        ("256_order", [(1025, 4096), (1280, 4096), (1281, 4096), (1536, 4097)], 2, "<256,4>", {True, False}),
        ("256_limit", [(1536, lim1536), (1200, 12000)], 2, "<256,4>", {False}),
        ("512_2", [(1537, 4096), (2560, 4096), (2561, 4096), (2000, 4095)], 2, "<512,2>", {True, False}),
        ("512_1", [(2000, 6000), (2561, 4097), (1537, 1)], 2, "<512,1>", {True, False}),
        ("512_largest_source", [(big, 1000), (2600, 1000)], 1, "<512,1>", {False}),
    ]


def _build(cases, k, seed0):
    pairs = []
    for j, (ns, nt) in enumerate(cases):
        s, t, T = _pair(ns, nt, seed0 + j)
        pairs.append((s, t, _guesses(T, k, seed0 + j)))
    return pairs


def _assert_class(pairs, cls, paths, plane=False, smid=None):
    ns_max, nt_max = max(len(p[0]) for p in pairs), max(len(p[1]) for p in pairs)
    d = dispatch(ns_max, nt_max, sum(len(p[2]) for p in pairs), plane)
    assert d["cls"] == cls, (d, cls)
    got = {one_pass(len(p[0]), len(p[1]), d["threads"]) for p in pairs}
    assert got == set(paths), (got, paths)
    if smid is not None:
        assert d["smid"] == smid, d
    return d


@pytest.mark.parametrize("checkers", list(CHECKERS))
@pytest.mark.parametrize("call", range(9))
def test_size_grid(gpu_ctx, call, checkers):
    name, cases, k, cls, paths = _size_calls()[call]
    pairs = _build(cases, k, 100 * call)
    d = _assert_class(pairs, cls, paths)
    if name.endswith("limit"):
        assert d["trimmed"] and max(len(p[1]) for p in pairs) == cta_limit(max(len(p[0]) for p in pairs))
    if "order" in name or name.startswith("512"):
        assert d["order"]
    prm, oprm = _params(**CHECKERS[checkers])
    _, wants = check_pairs(pairs, prm, oprm, name)
    assert sum(w["status"] == 0 for ws in wants for w in ws) >= len(pairs)


@pytest.mark.parametrize("threads,ns,nt", [(128, 400, 12000), (256, 1500, 9000), (512, 2000, 6000)])
def test_one_cta_per_problem_slots_by_sm(gpu_ctx, threads, ns, nt):
    """More problems than SMs on layouts that allow one CTA per SM: one CTA per problem, workspace slot = SM id."""
    sms = _dev()[2]
    s, t, T = _pair(ns, nt, threads)
    gs = _guesses(T, sms + 9, threads, sd=(0.3, 0.3, 0.03))
    d = _assert_class([(s, t, gs)], dispatch(ns, nt, len(gs))["cls"], {False}, smid=True)
    assert d["threads"] == threads and d["per_sm"] == 1
    prm, oprm = _params(**FIXED20)
    res = _icp(prm).compute_batch(s, t, gs)
    for k, g in enumerate(gs):
        _assert_equal(res, k, s, t, g, oprm, "smid")


@pytest.mark.parametrize("call,knn", [(0, 3), (1, 5), (4, 16), (6, 5), (7, 3)])
def test_point_to_plane_per_class(gpu_ctx, call, knn):
    name, cases, k, cls, paths = _size_calls()[call]
    cases = [(ns, nt) for ns, nt in cases if ns >= 3 and nt >= 16]  # normals need a neighbourhood
    pairs = _build(cases, 1, 100 * call)
    _assert_class(pairs, cls, {one_pass(ns, nt, icp_threads(max(c[0] for c in cases))) for ns, nt in cases},
                  plane=True)
    prm, oprm = _params(minimizer=1, normals_knn=knn, **FIXED20)
    check_pairs(pairs, prm, oprm, name + "_plane")


# ------------------------------------------------------------------ settings grid
SETTINGS = (
    [("matcher_" + str(m), dict(matcher_max_dist=m)) for m in (float("inf"), 1e9, 0.3, 10.0)]
    + [("outlier_off", dict(outlier_max_dist=-1.0)), ("outlier_sq", dict(outlier_max_dist=2.0, trim_ratio=-1.0)),
       ("outlier_raw", dict(outlier_max_dist=2.0, trim_ratio=-1.0, flags=1)),
       ("outlier_raw_trim", dict(outlier_max_dist=2.0, flags=1))]
    + [("trim_" + str(r), dict(trim_ratio=r)) for r in (-1.0, 1.0, 0.0, 0.5, 0.95)]
    + [("trim_off_inf", dict(trim_ratio=-1.0, matcher_max_dist=float("inf"))),
       ("trim_1_inf", dict(trim_ratio=1.0, matcher_max_dist=float("inf"), outlier_max_dist=-1.0))]
    + [("smooth_" + str(s), dict(smooth_length=s, max_iterations=40, min_diff_rot=0.0, min_diff_trans=0.0))
       for s in (1, 4, 15)]
    + [("huge_min_diff", dict(min_diff_rot=1e9, min_diff_trans=1e9)), ("one_iteration", dict(max_iterations=1))]
)
# (ns, nt) per thread count x path; "map": 1 000 points of the 30 000-point map of test_map_icp_gpu
SHAPES = {"128_onepass": (400, 1500), "128_pruned": (400, 12000), "256_onepass": (1000, 3000),
          "256_pruned": (1400, 6000), "512_onepass": (2000, 4000), "512_pruned": (2000, 20000), "map": None}


def _map30k():
    return orc.downsample(synth.make_map_cloud(400000, seed=11)[0], 0.1)[0][:30000]


_SHAPE_CACHE = {}


def _shape(name):
    if name not in _SHAPE_CACHE:
        if name == "map":
            tgt = _map30k()
            rng = np.random.default_rng(3)
            c = tgt[rng.integers(len(tgt))]
            near = tgt[np.linalg.norm(tgt - c, axis=1) < 30.0]
            src = near[rng.choice(len(near), min(1000, len(near)), replace=False)]
            T = synth.se2(c[0] + 1.0, c[1] - 1.0, 0.4)
            Ti = np.linalg.inv(T)
            src = np.concatenate([src @ Ti[:2, :2].T + Ti[:2, 2], rng.uniform(-40, 40, (200, 2))]).astype(F32)
            _SHAPE_CACHE[name] = (src, tgt, _guesses(T, 2, 3))
        else:
            ns, nt = SHAPES[name]
            s, t, T = _pair(ns, nt, 7000 + ns + nt)
            _SHAPE_CACHE[name] = (s, t, _guesses(T, 2, ns))
    return _SHAPE_CACHE[name]


@pytest.mark.parametrize("shape", list(SHAPES))
def test_settings_grid(gpu_ctx, shape):
    s, t, gs = _shape(shape)
    d = dispatch(len(s), len(t), len(gs))
    if shape == "map":
        assert d["cls"] == "map"
    else:
        assert d["threads"] == int(shape[:3]) and one_pass(len(s), len(t), d["threads"]) == shape.endswith("onepass")
    inl = {}
    for name, kw in SETTINGS:
        prm, oprm = _params(**kw)
        res = _icp(prm).compute_batch(s, t, gs)
        wants = [_assert_equal(res, k, s, t, g, oprm, (shape, name)) for k, g in enumerate(gs)]
        inl[name] = [w["inliers"] for w in wants]
        if name == "huge_min_diff":
            assert all(w["iterations"] == 4 for w in wants if w["status"] == 0)  # the first differential check
        if name == "one_iteration":
            assert all(w["iterations"] == 1 for w in wants if w["status"] == 0)
        if name == "smooth_15":
            assert any(w["iterations"] == 40 for w in wants)  # past the 16-entry history: it shifted
    assert inl["outlier_raw"] != inl["outlier_sq"], inl  # raw vs squared 2.0 keep different sets


def test_config3_pair_without_matcher_max_dist(gpu_ctx):
    """A config-3 pair (2 000 x 20 000, 20 % of the source far from every wall) with the matcher's maxDist removed
    (libpointmatcher's default: inf).  The far outliers reach pass B of the pruned path; the oracle matches them all."""
    s, t, _ = synth.make_icp_pair(3)
    assert dispatch(len(s), len(t), 1)["cls"] == "<512,1>" and not one_pass(len(s), len(t), 512)
    for kw in (dict(matcher_max_dist=float("inf")), dict(matcher_max_dist=1e9), dict(matcher_max_dist=3e19)):
        for chk in CHECKERS.values():
            prm, oprm = _params(**kw, **chk)
            res = _icp(prm).compute_batch(s, t, [np.eye(3, dtype=F32)])
            w = _assert_equal(res, 0, s, t, np.eye(3, dtype=F32), oprm, kw)
            assert w["status"] == 0


# ------------------------------------------------------------------ knife-edge geometry
def lattice(k):
    a = np.arange(-k, k + 1, dtype=np.float64)
    return np.array(list(itertools.product(a, a)), F32)


def knife_source(k, offsets, seed, n_each):
    rng = np.random.default_rng(seed)
    out = [rng.integers(-k + 2, k - 1, size=(n_each, 2)).astype(np.float64) + np.asarray(o) for o in offsets]
    s = np.concatenate(out).astype(F32)
    return s[rng.permutation(len(s))]


def _brute_d2(src, tgt):
    dx = src[:, None, 0] - tgt[None, :, 0]
    dy = src[:, None, 1] - tgt[None, :, 1]
    return dx * dx + dy * dy  # float32, unfused


@pytest.mark.parametrize("path,k", [("onepass", 20), ("pruned", 40)])
def test_knife_edges(gpu_ctx, path, k):
    tgt = lattice(k)[np.random.default_rng(k).permutation((2 * k + 1) ** 2)]
    src = knife_source(k, [(0.5, 0.0), (0.0, 0.5), (0.5, 0.5), (0.25, 0.0), (0.0, 0.125)], k, 110)
    assert np.cumsum(tgt, axis=0, dtype=F32)[-1].tolist() == [0.0, 0.0]  # the oracle's centring is exact
    d = dispatch(len(src), len(tgt), 1)
    assert one_pass(len(src), len(tgt), d["threads"]) == (path == "onepass")
    d2 = _brute_d2(src, tgt)
    dmin = d2.min(1)
    n_min = (d2 == dmin[:, None]).sum(1)
    # the edges this case claims: points at exactly 0.5 m (d2 0.25) and at d2 0.5, 2- and 4-way ties, the lowest
    # index not first in the lattice's row-major order, many equal distances
    assert (dmin == F32(0.25)).sum() >= 200 and (dmin == F32(0.5)).sum() >= 100
    assert (n_min == 2).sum() >= 200 and (n_min == 4).sum() >= 100
    first = np.array([min(np.flatnonzero(r == r.min()), key=lambda j: (tgt[j, 1], tgt[j, 0])) for r in d2])
    assert (first != np.argmin(d2, 1)).sum() >= 100
    one = dict(max_iterations=1, smooth_length=0)
    settings = [dict(matcher_max_dist=0.5, outlier_max_dist=-1.0, trim_ratio=-1.0),   # d2 == maxDist^2 accepted
                dict(outlier_max_dist=0.5, trim_ratio=-1.0),                           # squared MaxDist edge
                dict(outlier_max_dist=0.5, trim_ratio=-1.0, flags=1),                  # raw MaxDist edge (d2 = 0.5)
                dict(outlier_max_dist=-1.0, trim_ratio=0.5),                           # quantile among equal distances
                dict(outlier_max_dist=-1.0, trim_ratio=0.95),
                dict(outlier_max_dist=-1.0, trim_ratio=0.0),
                dict(outlier_max_dist=-1.0, trim_ratio=-1.0),                          # ties decide the fit
                dict(matcher_max_dist=float("inf"), outlier_max_dist=-1.0, trim_ratio=0.5)]
    inliers = []
    for kw in settings:
        prm, oprm = _params(**kw, **one)
        res = _icp(prm).compute_batch(src, tgt, [np.eye(3, dtype=F32)])
        w = _assert_equal(res, 0, src, tgt, np.eye(3, dtype=F32), oprm, kw)
        inliers.append(w["inliers"])
    fin = dmin <= F32(0.25)
    assert inliers[0] == fin.sum()
    assert inliers[1] == (dmin <= F32(0.25)).sum() and inliers[2] == (dmin <= F32(0.5)).sum() > inliers[1]
    s = np.sort(dmin)
    assert (dmin == s[int(F32(len(s)) * F32(0.5))]).sum() >= 200  # the quantile element has many equals


# ------------------------------------------------------------------ degenerate targets
def _degenerate(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "collinear":
        t = np.c_[rng.uniform(-20, 20, n), np.full(n, 3.0)]
    elif kind == "identical":
        t = np.tile([[3.0, 4.0]], (n, 1))
    elif kind == "duplicated":
        h = _pair(10, n // 2, seed)[1]
        t = np.concatenate([h, h[::-1]])
    elif kind == "corridor":
        t = np.c_[rng.uniform(0, 3000, n), rng.uniform(-0.25, 0.25, n)]
    elif kind == "far_point":
        t = _pair(10, n - 1, seed)[1]
        t = np.concatenate([t[: n // 2], [[1e4, 0.0]], t[n // 2:]])
    elif kind == "offset":
        t = _pair(10, n, seed)[1] + 1e4
    else:  # 1 mm extent
        t = rng.uniform(0, 1e-3, (n, 2)) + [2.0, -1.0]
    t = t.astype(F32)
    pick = t[rng.choice(n, min(500, n), replace=False)].astype(np.float64)
    scale = 1e-4 if kind == "mm" else 0.05
    src = (pick + rng.normal(0, scale, pick.shape)).astype(F32)
    rot = 0.0 if kind in ("mm", "offset") else 0.01  # (a turn about the origin would move a cloud 10 km out by 100 m)
    return src, t, [np.eye(3, dtype=F32), synth.se2(scale, -scale, rot).astype(F32)]


@pytest.mark.parametrize("kind", ["collinear", "identical", "duplicated", "corridor", "far_point", "offset", "mm"])
def test_degenerate_targets(gpu_ctx, kind):
    sizes = (12000,) if kind == "corridor" else (3000, 6000)
    for n in sizes:
        src, tgt, gs = _degenerate(kind, n, n)
        d = dispatch(len(src), len(tgt), len(gs))
        assert one_pass(len(src), len(tgt), d["threads"]) == (n <= 4096)
        if kind == "corridor":
            # a coarse map hundreds of cells long and one high.  Its skip above 96 * 32 coarse cells cannot be
            # reached by an in-CTA target: a cell table of at most 16 384 cells makes at most 2 048 coarse cells
            mc = layout(len(src), len(tgt))[1]
            assert 500 <= coarse_cells(tgt, mc) <= GRID_MAX_CELLS // 8 < COARSE_WORDS * 32
        for chk in CHECKERS.values():
            prm, oprm = _params(**chk)
            res = _icp(prm).compute_batch(src, tgt, gs)
            for k, g in enumerate(gs):
                _assert_equal(res, k, src, tgt, g, oprm, (kind, n))


# ------------------------------------------------------------------ the user's route, and what it must refuse
USER_YAML = """matcher:
  KDTreeMatcher:
    knn: 1
    epsilon: 0
outlierFilters:
  - MaxDistOutlierFilter:
      maxDist: 2.0
  - TrimmedDistOutlierFilter:
      ratio: 0.95
errorMinimizer:
  PointToPointErrorMinimizer
transformationCheckers:
  - CounterTransformationChecker:
      maxIterationCount: 30
  - DifferentialTransformationChecker:
      minDiffRotErr: 0.001
      minDiffTransErr: 0.01
      smoothLength: 6
"""


def test_user_yaml_through_pcl_icp(gpu_ctx, tmp_path):
    from sonar_slam_b200.bruce_slam import pcl
    p = tmp_path / "icp.yaml"
    p.write_text(USER_YAML)
    icp = pcl.ICP()
    icp.loadFromYaml(str(p))
    assert icp.params.matcher_max_dist == float("inf") and icp.params.smooth_length == 6
    oprm = _oracle_params(icp.params)
    for ns, nt, seed in ((400, 1500, 1), (400, 12000, 2), (2000, 20000, 3)):
        s, t, T = _pair(ns, nt, 8000 + seed)
        gs = _guesses(T, 3, seed)
        res = icp.compute_batch(s, t, gs)
        for k, g in enumerate(gs):
            _assert_equal(res, k, s, t, g, oprm, ("yaml", ns, nt))


@pytest.mark.parametrize("kw", [dict(trim_ratio=1.5), dict(trim_ratio=float("nan")),
                                dict(matcher_max_dist=float("nan")), dict(outlier_max_dist=float("nan")),
                                dict(min_diff_rot=float("nan")), dict(min_diff_trans=float("nan"))])
def test_icp_run_rejects_settings_before_any_launch(gpu_ctx, kw):
    from sonar_slam_b200 import _lib
    ctx = _lib.default_context()
    s, t, T = _pair(300, 1000, 9)
    prm, _ = _params(**kw)
    n0 = ctx.launches
    with pytest.raises(_lib.SonarFEError):
        _icp(prm).compute_batch(s, t, [T.astype(F32)])
    assert ctx.launches == n0
