"""GPU: the persistent kernels hold to the oracles on every work item, not only on each CTA's first.

Persistent CTAs take item after item from a work counter or by striding, and carry state across items on purpose
(zeroed histograms, rotation counters, per-CTA workspace slices, shared tables rewritten per item).  A full-size grid
gives most CTAs one item, so these tests run every such launch on a context capped at one SM
(sfe_ctx_set_grid_sms): 1 to 8 CTAs, each taking tens of items in a row.  Batches are laid out so that every kind of
item (empty, one point, coincident points, deep trees, over capacity, every ICP exit ...) directly follows every other
kind, and are also run in two seeded permutations.  Every output of every item must equal the CPU oracle bit for bit
and the same batch on the uncapped context.  The last test runs a bag with more frames than one wave of the front
end's small ICP class on the uncapped context and holds every frame to the capped run and the oracle chain."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import cloud3_ref as c3
from oracle import featx_ref, knn_ref, pipeline_ref
from oracle import icp3_ref as o3
from oracle import octree_filter_ref as ofr
from oracle import oracle as orc
from oracle import voxel_filter_ref as vfr
from sonar_slam_b200 import _lib, ops, pipeline, synth

pytestmark = pytest.mark.gpu

F32 = np.float32
TAU = 2.749063720096473
SMALL = (640, 800)      # pipeline.cu: FE_ICP_SMALL_SRC / _TGT, the front end's small ICP class
RO_CTA_LIMIT = 24445    # remove_outlier_kernel's largest cloud on an H100 (include/sonarfe.h); larger: the map class
MATCH_CTA_LIMIT = 24000  # below the one-CTA reference limit at knn 1 .. 2 (include/sonarfe.h); 30 000: the map grids
MX, MN, OCT, VOX = _lib.MAX_DIST, _lib.MIN_DIST, _lib.OCTREE, _lib.VOXEL


# ------------------------------------------------------------------ contexts and batch layout
@pytest.fixture(scope="module")
def ctxs(gpu_ctx):
    """(capped, uncapped): a context on torch's stream sized for one SM, and the session's full-size one."""
    dev_sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert gpu_ctx.set_grid_sms(0) == dev_sms
    capped = _lib.Context(0, torch.cuda.current_stream(0).cuda_stream)
    assert capped.set_grid_sms(10 ** 6) == dev_sms     # the cap never exceeds the device
    assert capped.set_grid_sms(1) == 1
    yield capped, gpu_ctx
    _lib.set_icp_filters(gpu_ctx, None)   # later modules share the session context
    capped.close()


def de_bruijn(k):
    """A sequence over 0 .. k-1 in which every ordered pair (a, b), a == b included, appears as neighbours."""
    seq, a = [], [0] * 2 * k

    def db(t, p):
        if t > 2:
            if 2 % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    return seq + seq[:1]


def layout(kinds, n):
    """n items: the kinds in de Bruijn order (repeated), so that each kind directly follows each other kind."""
    seq = de_bruijn(len(kinds))
    out = [kinds[seq[i % (len(seq) - 1)]] for i in range(n)]
    pairs = {(a, b) for a, b in zip(out, out[1:])}
    assert n < len(seq) or len(pairs) == len(kinds) ** 2
    return out


def perms(n):
    return [np.random.default_rng(seed).permutation(n) for seed in (1, 2)]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == F32 else a


def same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and np.array_equal(_bits(a), _bits(b)), what


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def pack(clouds, dim=2):
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    pts = np.concatenate([np.asarray(c, F32).reshape(-1, dim) for c in clouds] + [np.zeros((0, dim), F32)])
    return _dev(pts), _dev(off), off


def _host(d):
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in d.items()}


# ------------------------------------------------------------------ Cartesian points
def test_cart_points_every_frame(ctxs):
    capped, full = ctxs
    geo = featx_ref.Geometry(30.0 / 512, 512, synth.bearings_oculus(512))
    maps = _lib.Maps(full, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    rng = np.random.default_rng(0)
    kinds = layout(["blank", "sparse", "dense", "over"], 200)
    density = dict(blank=0.0, sparse=0.002, dense=0.05, over=0.2)
    masks = np.stack([(rng.random((512, 512)) < density[k]).astype(np.uint8) for k in kinds])
    want = [featx_ref.cart_points(m, geo) for m in masks]
    counts = np.array([len(w[0]) for w in want])
    over = np.array([k == "over" for k in kinds])
    cap = int(counts[~over].max())                 # the largest frame below capacity fills it exactly
    assert (counts[over] > cap).all() and (counts[np.array(kinds) == "blank"] == 0).all()
    bits = np.packbits(masks, axis=-1, bitorder="little").view(np.uint32).view(np.int32)

    def check(out, order, what):
        got = _host(out)
        same(got["count"], counts[order], what)
        for j, f in enumerate(order):
            k = min(counts[f], cap)
            same(got["ij"][j, :k], want[f][0][:k], (what, j, kinds[f]))
            same(got["xy"][j, :k], want[f][1][:k].astype(F32), (what, j, kinds[f]))
        return got

    ident = np.arange(len(kinds))
    for name, src in (("mask", masks), ("bits", bits)):
        a = check(ops.cart_points(maps, capacity=cap, ctx=capped, **{name: _dev(src)}), ident, (name, "capped"))
        b = check(ops.cart_points(maps, capacity=cap, ctx=full, **{name: _dev(src)}), ident, (name, "full"))
        for k in a:
            same(a[k], b[k], (name, k))
        for order in perms(len(kinds)):
            check(ops.cart_points(maps, capacity=cap, ctx=capped, **{name: _dev(src[order])}), order, (name, "perm"))


# ------------------------------------------------------------------ down-sample
def _walls(rng, n, dim, extent=40.0):
    if n == 0:
        return np.zeros((0, dim), F32)
    p = synth.sample_walls(rng, synth.make_walls(rng, n_segments=6, extent=extent), n, 0.05)
    if n > 10:
        p[: n // 5] = rng.uniform(0, extent, (n // 5, 2))
    if dim == 3:
        p = np.c_[p, rng.normal(0, 0.3, n)]
    return p.astype(F32)


def _cloud(kind, rng, dim, res, sizes):
    if kind == "empty":
        return np.zeros((0, dim), F32)
    if kind == "one":
        return rng.uniform(-5, 5, (1, dim)).astype(F32)
    if kind == "coincident":
        return np.repeat(rng.uniform(-5, 5, (1, dim)).astype(F32), int(rng.integers(2, 300)), 0)
    if kind == "deep":   # two blobs 2^17 resolutions apart: more than 15 levels below the root
        blob = rng.uniform(0, 6 * res, (int(rng.integers(20, 60)), dim))
        return np.concatenate([blob, blob[: len(blob) // 2] + 2.0 ** 17 * res]).astype(F32)
    lo, hi = sizes
    return _walls(rng, int(rng.integers(lo, hi + 1)), dim)


def _ds_want(cl, kind, dim, res):
    """(points, indices) of the oracle; clouds deeper than 15 levels against the trees cut there, as the device's."""
    if dim == 3:
        if kind == "deep":
            idx = c3.octree_literal(cl, res, max_depth=15)
            return cl[idx], idx
        return c3.downsample3(cl, res)
    if kind == "deep":
        return ofr.octree_filter(cl, res, 3, max_depth=15), None
    return orc.downsample(cl, res)


def _ds_check(got, clouds, kinds, off_h, wants, order, what):
    for j, c in enumerate(order):
        wp, wi = wants[c]
        s, k = off_h[j], int(got["count"][j])
        assert k == len(wp), (what, j, kinds[c], k, len(wp))
        same(got["pts"][s:s + k], wp, (what, j, kinds[c]))
        if wi is not None:
            same(got["idx"][s:s + k], wi.astype(np.int32), (what, j, kinds[c]))
        else:      # the cut 2-D tree's medoids: the indices name them
            same(clouds[c][got["idx"][s:s + k]], wp, (what, j, kinds[c]))


# (name, dim, entry point, cloud sizes of the "walls" kind, frame_points of the front end's launch or None)
DS_CASES = {
    "2d_256_threads": (2, (100, 2048), None),
    "2d_512_threads": (2, (1500, 6000), None),
    "2d_cta_and_grid": (2, (3000, 16000), None),
    "2d_frames_global_ws": (2, (1500, 16000), 2048),
    "3d_256_threads": (3, (100, 2048), None),
    "3d_cta_and_grid": (3, (1500, 12000), None),
}


@pytest.mark.parametrize("case", list(DS_CASES))
def test_downsample_every_cloud(ctxs, case):
    capped, full = ctxs
    dim, sizes, frame_points = DS_CASES[case]
    rng = np.random.default_rng(sum(map(ord, case)))
    kinds = layout(["empty", "one", "coincident", "deep", "walls"], 40 if sizes[1] > 6000 else 60)
    limit = ops.downsample_cta_limit(dim, ctx=full)
    if sizes[1] > 6000:     # sizes on both sides of the one-CTA limit, one of them exactly at it
        assert sizes[0] < limit < sizes[1]
    for res in (0.5, 0.13, 7.0):
        clouds = [_cloud(k, rng, dim, res, sizes) for k in kinds]
        if sizes[1] > 6000:
            clouds[kinds.index("walls")] = _walls(rng, limit, dim)
        if sizes[1] == 2048:
            clouds[kinds.index("walls")] = _walls(rng, 2048, dim)
        n_max = max(len(c) for c in clouds)
        wants = [_ds_want(c, k, dim, res) for c, k in zip(clouds, kinds)]

        def run(ctx, order):
            cl = [clouds[c] for c in order]
            pts, off, off_h = pack(cl, dim)
            if frame_points is None:
                out = ops.downsample(pts, off, n_max, res, ctx=ctx)
            else:
                out = ops.downsample_frames(pts, off, n_max, res, frame_points, ctx=ctx)
            got = _host(out)
            _ds_check(got, clouds, kinds, off_h, wants, order, (case, res))
            return got

        ident = np.arange(len(clouds))
        a, b = run(capped, ident), run(full, ident)
        for k in a:
            same(a[k], b[k], (case, res, k))
        for order in perms(len(clouds)):
            run(capped, order)


# ------------------------------------------------------------------ outlier removal
@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("klass", ["cta", "map"])
def test_remove_outlier_every_cloud(ctxs, dim, klass):
    capped, full = ctxs
    rng = np.random.default_rng(10 * dim + (klass == "map"))
    kinds = layout(["empty", "one", "coincident", "small", "large"], 40)
    clouds, n_big = [], 0
    for k in kinds:
        if k == "small":
            clouds.append(_walls(rng, int(rng.integers(10, 1024)), dim))
        elif k == "large":   # the map class: three clouds above the one-CTA limit, the rest of this kind below it
            n = int(rng.integers(RO_CTA_LIMIT + 1, RO_CTA_LIMIT + 2000)) if klass == "map" and n_big < 3 else \
                int(rng.integers(3000, 9000))
            n_big += n > RO_CTA_LIMIT
            clouds.append(_walls(rng, n, dim, extent=60.0))
        else:
            clouds.append(_cloud(k, rng, dim, 0.5, None))
    assert n_big == (3 if klass == "map" else 0)
    n_max = max(len(c) for c in clouds)
    for radius, mp in ((0.3, 1), (2.5, 40)):
        wants = [orc.remove_outlier(c, radius, mp) if len(c) else (c, np.zeros(0, bool)) for c in clouds]

        def run(ctx, order):
            pts, off, off_h = pack([clouds[c] for c in order], dim)
            got = _host(ops.remove_outlier(pts, off, n_max, radius, mp, ctx=ctx))
            for j, c in enumerate(order):
                wp, keep = wants[c]
                s, k = off_h[j], int(got["count"][j])
                assert k == len(wp), (dim, klass, radius, j, kinds[c])
                same(got["pts"][s:s + k], wp, (dim, klass, radius, j))
                same(got["idx"][s:s + k], np.nonzero(keep)[0].astype(np.int32), (dim, klass, radius, j))
            return got

        ident = np.arange(len(clouds))
        a, b = run(capped, ident), run(full, ident)
        for k in a:
            same(a[k], b[k], (dim, klass, radius, k))
        for order in perms(len(clouds)):
            run(capped, order)


# ------------------------------------------------------------------ match
def _match_want(ref, q, knn, md, dim):
    if dim == 3:
        return c3.match_knn3(ref, q, knn or 1, md)
    if knn is None:
        return orc.match(ref, q, md)
    return knn_ref.match_knn(ref, q, knn, md)


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("klass", ["cta", "map"])
@pytest.mark.parametrize("knn", [None, 2, 16])
def test_match_every_pair(ctxs, dim, klass, knn):
    capped, full = ctxs
    rng = np.random.default_rng(100 * dim + 7 * (knn or 1) + (klass == "map"))
    kinds = layout(["empty", "one", "coincident", "small", "large"], 30)
    refs, qs = [], []
    n_big = 0
    for k in kinds:
        if k == "large":
            n = 30000 if klass == "map" and n_big < 2 else int(rng.integers(2000, 6000))
            n_big += n == 30000
            r = rng.uniform(0, 60, (n, dim)).astype(F32)
        elif k == "small":
            r = rng.uniform(0, 8, (int(rng.integers(5, 500)), dim)).astype(F32)
        else:
            r = _cloud(k, rng, dim, 0.5, None)
        refs.append(r)
        span = 60 if k == "large" else 8
        qs.append(rng.uniform(-0.2 * span, 1.2 * span, (int(rng.integers(0, 400)), dim)).astype(F32))
    assert klass == "cta" or n_big == 2
    n_ref_max = max(len(r) for r in refs)
    assert (n_ref_max > MATCH_CTA_LIMIT) == (klass == "map")
    for md in (0.5, 10.0):
        wants = [_match_want(r, q, knn, md, dim) for r, q in zip(refs, qs)]

        def run(ctx, order):
            rp, ro, _ = pack([refs[c] for c in order], dim)
            ip, io, io_h = pack([qs[c] for c in order], dim)
            got = _host(ops.match(rp, ro, ip, io, n_ref_max, md, knn=knn, ctx=ctx))
            for j, c in enumerate(order):
                s, e = io_h[j], io_h[j + 1]
                wi, wd = wants[c]
                gi, gd = (got["ids"][s:e], got["dists"][s:e]) if knn is None else \
                    (got["ids"][:, s:e], got["dists"][:, s:e])
                same(gi, wi[0] if knn is None else wi, (dim, klass, knn, md, j, kinds[c]))
                same(gd, wd[0] if knn is None else wd, (dim, klass, knn, md, j, kinds[c]))
            return got

        ident = np.arange(len(refs))
        a, b = run(capped, ident), run(full, ident)
        for k in a:
            same(a[k], b[k], (dim, klass, knn, md, k))
        for order in perms(len(refs)):
            run(capped, order)


# ------------------------------------------------------------------ ICP through ops.icp
def _top_up(t, n, rng, dim):
    if len(t) >= n:
        return np.ascontiguousarray(t[:n], F32)
    extra = t[rng.integers(len(t), size=n - len(t))] + rng.normal(0, 0.03, (n - len(t), dim))
    return np.concatenate([t, extra]).astype(F32)


def _far(dim):
    g = np.eye(dim + 1, dtype=F32)
    g[:2, dim] = 100.0
    return g


def _icp_problem(kind, seed, dim, ns_big):
    """(source, target, guess) of one ICP work item of `kind`."""
    rng = np.random.default_rng(seed)
    # large: the largest layout of the in-CTA batches, with room for two CTAs per SM (a 3-D CTA laid out for 1 500 / 6 000
    # points takes 126 KB of shared memory: one per SM, and that launch runs one CTA per problem)
    large = (1500, 6000) if dim == 2 else (1200, 3500)
    ns, nt = dict(small=(int(rng.integers(60, 200)), int(rng.integers(120, 400))), large=large,
                  gsrc=(ns_big, 3000)).get(kind, (int(rng.integers(100, 600)), 900))
    if kind.startswith("map"):   # above the one-CTA target limit next to sources of up to 1 500 points
        ns, nt = int(rng.integers(200, 600)), int(rng.integers(23000, 26000))
        kind = kind[4:]
    if dim == 2:
        s, t, T = synth.make_icp_pair(seed, n_source=ns, n_target=min(nt, 20000))
        T = np.asarray(T, np.float64) @ synth.se2(*rng.normal(0, (0.2, 0.2, 0.02)))
    else:
        s, t, T = synth.make_icp_pair3(seed, n_source=ns, n_target=nt)
        T = np.asarray(T, np.float64) @ synth.se3(rng.normal(0, 0.2, 3), rng.normal(size=3), rng.normal(0, 0.02))
    s, t, g = _top_up(s, ns, rng, dim), _top_up(t, nt, rng, dim), T.astype(F32)
    if kind == "far":        # no source point within maxDist: NO_OUTLIER (NO_POINT without the trimmed filter)
        g = _far(dim)
    elif kind == "not_rigid":
        g = g.copy()
        g[0, 0] *= 1.2
    elif kind == "empty_tgt":
        t = np.zeros((0, dim), F32)
    elif kind == "empty_src":
        s = np.zeros((0, dim), F32)
    return s, t, g


FIXED20 = dict(max_iterations=20, smooth_length=0)
ICP_SETTINGS = {  # name: (IcpParams keywords, IcpFilters keywords or None)
    "checkers": ({}, None),
    "cap40": (dict(min_diff_rot=1e-9, min_diff_trans=1e-9), None),
    "fixed20": (FIXED20, None),
    "no_trim": (dict(trim_ratio=-1.0), None),
    "plane": (dict(minimizer=1, normals_knn=5), None),
    "distance": ({}, dict(min_dist=0.05, reading=[(MX, -1, 18.0)], reference=[(MN, 0, -30.0)])),
    "median": (dict(trim_ratio=-1.0, **FIXED20), dict(median_factor=1.5)),   # the only quantile filter
    "octree": ({}, dict(reading=[(OCT, 2, 0.3)], reference=[(OCT, 3, 0.2)])),
    "voxel": ({}, dict(reading=[(VOX, 1, 0.25)], reference=[(VOX, 1, 0.2)])),
    "3d": ({}, None),
}
# the exit each kind must take under the oracle (a set where several are allowed)
EXITS = {"small": {0, 2}, "large": {0}, "map": {0}, "gsrc": {0}, "not_rigid": {5}, "empty_tgt": {6}, "map_not_rigid": {5}}


def expected_exits(kind, setting):
    """A source with no point within maxDist ("far") or no point at all: NO_OUTLIER (1) while a quantile filter
    (TrimmedDist, or MedianDist with no finite distance) is on, NO_POINT (2) without one."""
    if kind in ("far", "map_far", "empty_src"):
        return {2} if setting == "no_trim" else {1}
    return EXITS[kind]


def _icp_want(probs, setting, dim):
    kw, fkw = ICP_SETTINGS[setting]
    prm = orc.IcpParams(**kw)
    if dim == 3:
        return o3.icp3_many(probs, prm)
    if fkw is None:
        return [orc.icp(s, t, g, prm) for s, t, g in probs]
    return [vfr.icp(s, t, g, prm, vfr.IcpFilters(**fkw)) for s, t, g in probs]


def _icp_run(ctx, probs, setting, dim, order):
    kw, fkw = ICP_SETTINGS[setting]
    sp, so, _ = pack([probs[c][0] for c in order], dim)
    tp, to, _ = pack([probs[c][1] for c in order], dim)
    g = _dev(np.stack([probs[c][2] for c in order]))
    ns, nt = max(len(p[0]) for p in probs), max(len(p[1]) for p in probs)
    return _host(ops.icp(sp, so, tp, to, g, ns, nt, _lib.IcpParams(**kw), ctx=ctx,
                         filters=None if fkw is None else _lib.IcpFilters(**fkw)))


def _icp_check(got, want, kinds, order, what):
    for j, c in enumerate(order):
        w = want[c]
        row = (int(got["status"][j]), int(got["iterations"][j]), int(got["inliers"][j]))
        assert row == (w["status"], w["iterations"], w["inliers"]), (what, j, kinds[c], row, w)
        same(got["T"][j], np.asarray(w["T"], F32), (what, j, kinds[c]))


def fresh_capped():
    """A new context capped at one SM: its occupancy list then holds only the launches of the calls made on it."""
    ctx = _lib.Context(0, torch.cuda.current_stream(0).cuda_stream)
    assert ctx.set_grid_sms(1) == 1
    return ctx


def assert_several_per_cta(ctx, n_items, what):
    """Every persistent launch the calls on ctx sized runs at least 2 CTAs per SM, fewer than the items: at one SM a
    launch is then persistent (a layout with one CTA per SM would run the in-CTA ICP class one CTA per problem)."""
    occ = ctx.occupancy()
    assert occ and all(2 <= q < n_items for _, _, q in occ), (what, occ)


def _icp_batch(ctxs, setting, dim, kinds, seed0, ns_big=0, several_per_sm=False):
    capped, full = ctxs
    probs = [_icp_problem(k, seed0 + 13 * j, dim, ns_big) for j, k in enumerate(kinds)]
    want = _icp_want(probs, setting, dim)
    for k, w in zip(kinds, want):   # each kind takes the exit it was built for
        assert w["status"] in expected_exits(k, setting), (setting, k, w["status"])
    ident = np.arange(len(probs))
    one = fresh_capped()
    a = _icp_run(one, probs, setting, dim, ident)
    if several_per_sm:
        assert_several_per_cta(one, len(probs), setting)
    one.close()
    _icp_check(a, want, kinds, ident, (setting, "capped"))
    b = _icp_run(full, probs, setting, dim, ident)
    for k in a:
        same(a[k], b[k], (setting, k))
    for order in perms(len(probs)):
        _icp_check(_icp_run(capped, probs, setting, dim, order), want, kinds, order, (setting, "perm"))
    return want


# The in-CTA launch is laid out for the call's largest target up to the one-CTA limit: a batch without map-sized targets
# keeps that layout small, so several persistent CTAs share the problems (a layout that fills the SM runs one CTA per
# problem instead; the in-CTA batches check it).  The map batch sends most problems to the map class, whose CTAs are
# persistent at any occupancy, as are the global-source class's.
ICP_KINDS = {"cta": ["small", "large", "far", "not_rigid", "empty_tgt", "empty_src"],
             "map": ["map", "map_far", "map_not_rigid", "small", "empty_tgt"]}
MAP_SETTINGS = ["checkers", "plane", "median", "3d"]


@pytest.mark.parametrize("klass,setting", [("cta", s) for s in ICP_SETTINGS] + [("map", s) for s in MAP_SETTINGS])
def test_icp_every_problem_in_cta_and_map_classes(ctxs, klass, setting):
    dim = 3 if setting == "3d" else 2
    kinds = layout(ICP_KINDS[klass], 40)
    want = _icp_batch(ctxs, setting, dim, kinds, seed0=1000 * len(setting) + (klass == "map"),
                      several_per_sm=klass == "cta")
    ok_iters = [w["iterations"] for k, w in zip(kinds, want) if w["status"] == 0]
    if setting in ("fixed20", "median"):
        assert set(ok_iters) == {20}
    elif setting == "cap40":   # the cap, and differential exits where a step is exactly zero
        assert 40 in ok_iters and len(set(ok_iters)) >= 2, ok_iters
    else:   # the differential checker ends problems at different iterations
        assert len(set(ok_iters)) >= 2, ok_iters


@pytest.mark.parametrize("dim", [2, 3])
def test_icp_every_problem_in_the_global_source_class(ctxs, dim):
    capped, full = ctxs
    S = ops.icp_source_limit(dim, ctx=full)
    assert 1536 < S < 65535
    kinds = layout(["gsrc", "far", "not_rigid", "empty_tgt"], 17)
    kinds += ["map"]    # a map-sized target: the call does not fit one CTA next to its sources
    _icp_batch(ctxs, "3d" if dim == 3 else "checkers", dim, kinds, seed0=77 + dim, ns_big=S + 1)


# ------------------------------------------------------------------ the front end's ICP classes
def _frontend_icp(ctx, probs, setting):
    P = len(probs)
    sp, so, _ = pack([p[0] for p in probs])
    tp, to, _ = pack([p[1] for p in probs])
    guess = _dev(np.stack([p[2] for p in probs]))
    T = torch.empty((P, 3, 3), dtype=torch.float32, device="cuda")
    iters, inl, st = (torch.empty(P, dtype=torch.int32, device="cuda") for _ in range(3))
    cls = torch.full((2 * P,), -1, dtype=torch.int32, device="cuda")
    prm = _lib.IcpParams(**ICP_SETTINGS[setting][0])
    p_ = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    _lib.set_icp_filters(ctx, None)
    _lib.check(ctx.lib.sfe_frontend_icp_dev(ctx.handle, ctypes.byref(prm), p_(sp), p_(so), p_(tp), p_(to), P,
                                            max(len(p[0]) for p in probs), max(len(p[1]) for p in probs), p_(guess),
                                            p_(T), p_(iters), p_(inl), p_(st), p_(cls)), "sfe_frontend_icp_dev")
    return _host(dict(T=T, iterations=iters, inliers=inl, status=st, cls=cls))


@pytest.mark.parametrize("setting", ["checkers", "plane"])
def test_frontend_icp_classes_every_problem(ctxs, setting):
    capped, full = ctxs
    kinds = layout(["tiny", "small_cls", "capacity", "far", "not_rigid", "empty_tgt"], 400)
    probs = []
    for j, k in enumerate(kinds):
        rng = np.random.default_rng(5000 + j)
        ns, nt = dict(tiny=(30, 50), small_cls=(int(rng.integers(300, 641)), int(rng.integers(400, 801))),
                      capacity=(int(rng.integers(641, 900)), int(rng.integers(700, 1200)))).get(k, (300, 500))
        s, t, g = _icp_problem("small", 5000 + j, 2, 0)
        s, t = _top_up(s, ns, rng, 2), _top_up(t, nt, rng, 2)
        if k == "far":
            g = _far(2)
        elif k == "not_rigid":
            g = g.copy()
            g[0, 0] *= 1.2
        elif k == "empty_tgt":
            t = np.zeros((0, 2), F32)
        probs.append((s, t, g))
    want = _icp_want(probs, setting, 2)
    assert {w["status"] for k, w in zip(kinds, want) if k in ("far", "not_rigid", "empty_tgt")} == {1, 5, 6}
    sizes = [(len(s), len(t)) for s, t, _ in probs]
    P = len(probs)

    def run(ctx, order):
        got = _frontend_icp(ctx, [probs[c] for c in order], setting)
        _icp_check(got, want, kinds, order, (setting, "frontend"))
        klass, place = got["cls"][:P], got["cls"][P:]     # every problem in one list, its class, largest first
        sz = [sizes[c] for c in order]
        assert klass.tolist() == [0 if a <= SMALL[0] and b <= SMALL[1] else 1 for a, b in sz]
        for c in range(2):
            members = np.flatnonzero(klass == c)
            assert sorted(place[members].tolist()) == list(range(len(members))), c
            ordered = members[np.argsort(place[members])]
            key = [(-min(sz[p][0] // 32, 31), p) for p in ordered]
            assert key == sorted(key), c
        return got

    ident = np.arange(P)
    one = fresh_capped()
    a, b = run(one, ident), run(full, ident)
    assert_several_per_cta(one, P, setting)   # both classes' launches
    one.close()
    assert (a["cls"][:P] == 0).sum() > 200 and (a["cls"][:P] == 1).sum() > 50
    for k in a:
        same(a[k], b[k], (setting, k))
    for order in perms(P):
        run(capped, order)


# ------------------------------------------------------------------ the fused front end
FE_MODES = {
    "checkers": ({}, None),
    "fixed20": (FIXED20, None),
    "plane": (dict(minimizer=1, normals_knn=5), None),
    "filters": ({}, dict(min_dist=0.05, reading=[(OCT, 2, 0.3)], reference=[(VOX, 1, 0.3)])),
}
# a resolution at which the matched frames fill both ICP classes, and capacities that hold their clouds
FE_KW = dict(resolution=0.35, submap_resolution=0.35, min_points=50, cap_source=4096, cap_target=12288)


def _fe(ctx, maps, n, mode, cap):
    kw, fkw = FE_MODES[mode]
    return pipeline.FrontEnd(ctx, maps, max_frames=n, icp=_lib.IcpParams(**kw), cap_points=cap, tau=TAU,
                             icp_filters=None if fkw is None else _lib.IcpFilters(**fkw), **FE_KW)


def _fe_want(frames, poses, geo, mode, cap):
    kw, fkw = FE_MODES[mode]
    return pipeline_ref.run(frames, poses, geo, icp_params=orc.IcpParams(**kw), cap_points=cap,
                            icp_filters=None if fkw is None else vfr.IcpFilters(**fkw), **FE_KW)


def _run_dev(fe, ctx, frames, poses):
    """run_dev over the whole bag (one call of every stage), its results read back like run_host's."""
    n = len(frames)
    dev = _dev(frames)
    pts, off = fe.run_dev(dev.data_ptr(), poses, n, clouds=True)
    r = fe.results_dev()
    got = dict(clouds=pts.cpu().numpy(), cloud_offsets=off.cpu().numpy(), T=ctx.to_host(r["T"], (n, 3, 3), F32),
               status=ctx.to_host(r["status"], (n,), np.int32), iterations=ctx.to_host(r["iterations"], (n,), np.int32),
               inliers=ctx.to_host(r["inliers"], (n,), np.int32))
    got["npoints"] = np.diff(got["cloud_offsets"]).astype(np.int32)
    return got


def _fe_check(got, clouds, want, what):
    same(got["npoints"], np.array([len(c) for c in clouds], np.int32), what)
    off = got["cloud_offsets"]
    for i, c in enumerate(clouds):
        same(got["clouds"][off[i]:off[i + 1]], c, (what, i))
        w = want[i]
        row = (int(got["status"][i]), int(got["iterations"][i]), int(got["inliers"][i]))
        assert row == (w["status"], w["iterations"], w["inliers"]), (what, i, row, w["status"])
        same(got["T"][i], np.asarray(w["T"], F32), (what, i))


@pytest.fixture(scope="module")
def fe_bag(ctxs):
    """64 frames: the trajectory bag with blank frames and frames whose detections are cut to a band (fewer than
    min_points), and a cloud capacity (cap_points) that at least 5 of its frames exceed."""
    n = 64
    d = synth.make_trajectory_frames(n, seed=21)
    frames, poses = d["frames"].numpy().copy(), d["poses_odom"]
    for i in range(n):
        if i % 9 == 4:
            frames[i] = 0
        elif i % 9 == 7:
            frames[i, :200] = 0
            frames[i, 230:] = 0
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(ctxs[1], geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    raw = np.array([pipeline_ref.frame_cloud_raw(f, geo, resolution=FE_KW["resolution"])[1] for f in frames])
    cap = int(np.sort(raw)[-7])
    assert cap > 1000 and (raw > cap).sum() >= 5 and (raw == 0).sum() >= 5, raw
    return frames, poses, geo, maps, cap


@pytest.mark.parametrize("mode", list(FE_MODES))
def test_fused_front_end_every_frame(ctxs, fe_bag, mode):
    capped, full = ctxs
    frames, poses, geo, maps, cap = fe_bag
    n = len(frames)
    clouds, want = _fe_want(frames, poses, geo, mode, cap)
    st = np.array([w["status"] for w in want])
    sizes = np.array([len(c) for c in clouds])
    assert (st == _lib.ICP_SKIPPED).sum() >= 8 and (st == _lib.ICP_TOO_LARGE).sum() >= 5 and (st == 0).sum() >= 20
    ok = st == 0
    assert (sizes[ok] > SMALL[0]).any() and (sizes[ok] <= SMALL[0]).any(), sizes[ok]  # both ICP classes hold frames
    fe = _fe(capped, maps, n, mode, cap)
    for chunk in (7, 64):
        _fe_check(fe.run_host(frames, poses, chunk_frames=chunk, clouds=True), clouds, want, (mode, chunk))
    _fe_check(_run_dev(fe, capped, frames, poses), clouds, want, (mode, "run_dev"))
    b = _fe(full, maps, n, mode, cap).run_host(frames, poses, chunk_frames=64, clouds=True)
    _fe_check(b, clouds, want, (mode, "full"))


def test_natural_scale_bag_past_one_wave(ctxs):
    """A bag with more frames than one wave of the small ICP class (8 CTAs per SM), on the uncapped context in one
    chunk (run_host) and in one call (run_dev): every stage runs once over the whole bag, so its persistent CTAs take
    more than one frame each.  Every frame equals the capped run and the oracle chain."""
    capped, full = ctxs
    wave = 8 * torch.cuda.get_device_properties(0).multi_processor_count
    n = int(wave * 1.1)
    d = synth.make_trajectory_frames(n, seed=33)
    frames, poses = d["frames"].numpy(), d["poses_odom"]
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(full, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    clouds, want = pipeline_ref.run(frames, poses, geo, cap_points=8192, cap_source=1024, cap_target=3072,
                                    threads=min(16, os.cpu_count() or 1))
    # the small class's one launch holds more problems than one wave of it: frames that reach ICP within its bounds
    small = [w["status"] not in (_lib.ICP_SKIPPED, _lib.ICP_TOO_LARGE) and len(c) <= SMALL[0]
             and w["n_target"] <= SMALL[1] for c, w in zip(clouds, want)]
    assert sum(small) > wave, (sum(small), wave)
    fe = pipeline.FrontEnd(full, maps, max_frames=n, tau=TAU)
    a = fe.run_host(frames, poses, chunk_frames=n, clouds=True)
    _fe_check(a, clouds, want, "natural scale, one chunk")
    _fe_check(_run_dev(fe, full, frames, poses), clouds, want, "natural scale, run_dev")
    b = pipeline.FrontEnd(capped, maps, max_frames=n, tau=TAU).run_host(frames, poses, chunk_frames=256, clouds=True)
    for k in a:
        same(a[k], b[k], k)
