"""Batch (device-resident) operator API over libsonarfe's *_dev entry points.

torch is used for what it is good at here -- owning device memory and streams; every
computation is a hand-written CUDA kernel inside libsonarfe.so.  All functions enqueue
on the torch current stream of the tensor's device and return torch tensors.
"""
import ctypes

import numpy as np
import torch

from . import _lib, _streams

ALG = {"CA": 0, "SOCA": 1, "GOCA": 2, "OS": 3}
_ctx_cache = {}


def context(device=None):
    """libsonarfe context bound to torch's current stream on `device`."""
    dev = torch.cuda.current_device() if device is None else torch.device(device).index or 0
    stream = torch.cuda.current_stream(dev).cuda_stream
    key = (dev, stream)
    ctx = _ctx_cache.get(key)
    if ctx is None:
        ctx = _ctx_cache[key] = _lib.Context(dev, stream)
    return ctx


def _dp(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def cfar(img, alg, train_hs, guard_hs, tau, k=0, gate=None, want_mask=True, want_thr=False, want_bits=False,
         ctx=None):
    """Batched CFAR (include/sonarfe.h: sfe_cfar_dev).

    img: cuda tensor [F, R, B] (or [R, B]) uint8 or float32, contiguous.
    Returns dict(mask=uint8[F,R,B] | None, thr=float32[F,R,B] | None, bits=int32[F,R,ceil(B/32)] | None).
    """
    if not img.is_cuda:
        raise _lib.SonarFEError("ops.cfar: image tensor must live on a CUDA device (no CPU path)")
    if img.dim() == 2:
        img = img.unsqueeze(0)
    if img.dtype not in (torch.uint8, torch.float32):
        raise TypeError("ops.cfar: image must be uint8 or float32")
    img = img.contiguous()
    F, R, B = img.shape
    ctx = ctx or context(img.device)
    mask = torch.empty((F, R, B), dtype=torch.uint8, device=img.device) if want_mask else None
    thr = torch.empty((F, R, B), dtype=torch.float32, device=img.device) if want_thr else None
    bits = torch.empty((F, R, (B + 31) // 32), dtype=torch.int32, device=img.device) if want_bits else None
    a = ALG[alg] if isinstance(alg, str) else int(alg)
    _lib.check(ctx.lib.sfe_cfar_dev(ctx.handle, _dp(img), 0 if img.dtype == torch.uint8 else 1, F, R, B, a,
                                    int(train_hs), int(guard_hs), int(k), float(tau),
                                    0 if gate is None else 1, 0.0 if gate is None else float(gate),
                                    _dp(mask), _dp(thr), _dp(bits)), "sfe_cfar_dev")
    return dict(mask=mask, thr=thr, bits=bits)


def cart_points(maps, mask=None, bits=None, capacity=8192, ctx=None):
    """Cartesian feature pixels / points of polar masks (include/sonarfe.h: sfe_cart_points_dev).

    maps: _lib.Maps.  mask: uint8 [F,R,B] cuda tensor, or bits: int32 [F,R,ceil(B/32)] (from cfar()).
    Returns dict(ij=int32[F,capacity,2], xy=float32[F,capacity,2], count=int32[F]).
    """
    src = mask if mask is not None else bits
    if src is None or not src.is_cuda:
        raise _lib.SonarFEError("ops.cart_points: pass a CUDA mask or bits tensor")
    if src.dim() == 2:
        src = src.unsqueeze(0)
    src = src.contiguous()
    F = src.shape[0]
    ctx = ctx or context(src.device)
    ij = torch.empty((F, capacity, 2), dtype=torch.int32, device=src.device)
    xy = torch.empty((F, capacity, 2), dtype=torch.float32, device=src.device)
    count = torch.empty((F,), dtype=torch.int32, device=src.device)
    _lib.check(ctx.lib.sfe_cart_points_dev(ctx.handle, maps.handle, _dp(src) if mask is not None else None,
                                           _dp(src) if mask is None else None, F, int(capacity), _dp(ij), _dp(xy),
                                           _dp(count)), "sfe_cart_points_dev")
    return dict(ij=ij, xy=xy, count=count)


def _offsets(counts, device):
    off = torch.zeros(len(counts) + 1, dtype=torch.int32, device=device)
    off[1:] = torch.cumsum(torch.as_tensor(counts, device=device), 0)
    return off


def downsample(pts, off, n_max, resolution, ctx=None):
    """Batched pcl.downsample on packed clouds (pts [total,2|3] f32, off [n+1] i32, cuda): the quadtree for 2 columns,
    the octree for 3."""
    ctx = ctx or context(pts.device)
    n = off.numel() - 1
    out = torch.empty_like(pts)
    idx = torch.empty((pts.shape[0],), dtype=torch.int32, device=pts.device)
    cnt = torch.empty((n,), dtype=torch.int32, device=pts.device)
    _lib.check(ctx.lib.sfe_downsample_dev(ctx.handle, _dp(pts), _dp(off), n, int(pts.shape[1]), int(n_max),
                                          float(resolution), _dp(out), _dp(idx), _dp(cnt)), "sfe_downsample_dev")
    return dict(pts=out, idx=idx, count=cnt)


def downsample_cta_limit(dim=2, ctx=None, device=0):
    """The largest cloud of `dim` columns downsample() runs in one CTA on this device (sfe_downsample_cta_limit);
    larger clouds take the grid-wide path."""
    ctx = ctx or context(device)
    out = np.zeros(1, np.int32)
    _lib.check(ctx.lib.sfe_downsample_cta_limit(ctx.handle, int(dim), _lib.ptr(out)), "sfe_downsample_cta_limit")
    return int(out[0])


def downsample_frames(pts, off, n_max, resolution, frame_points, cnt=None, ctx=None):
    """The front end's per-frame down-sample on packed clouds: clouds of up to `frame_points` points in a launch laid
    out for them, larger ones in a launch laid out for n_max <= 65535 (pts [total,2] f32, off [n+1] i32, optional cnt
    [n] i32, cuda).
    Same results as downsample()."""
    ctx = ctx or context(pts.device)
    n = off.numel() - 1
    out = torch.empty_like(pts)
    idx = torch.empty((pts.shape[0],), dtype=torch.int32, device=pts.device)
    count = torch.empty((n,), dtype=torch.int32, device=pts.device)
    _lib.check(ctx.lib.sfe_downsample_frames_dev(ctx.handle, _dp(pts), _dp(off), _dp(cnt) if cnt is not None else None,
                                                 n, int(n_max), int(frame_points), float(resolution), _dp(out),
                                                 _dp(idx), _dp(count)), "sfe_downsample_frames_dev")
    return dict(pts=out, idx=idx, count=count)


def remove_outlier(pts, off, n_max, radius, min_points, ctx=None):
    """Batched pcl.remove_outlier (include/sonarfe.h: sfe_remove_outlier_dev) on packed clouds (pts [total,2|3] f32, off
    [n+1] i32, cuda).  Clouds of any size: those above one CTA's shared memory (whole maps) run in the map class, a grid
    in global memory with one thread per point, with the same results."""
    ctx = ctx or context(pts.device)
    n = off.numel() - 1
    out = torch.empty_like(pts)
    idx = torch.empty((pts.shape[0],), dtype=torch.int32, device=pts.device)
    cnt = torch.empty((n,), dtype=torch.int32, device=pts.device)
    _lib.check(ctx.lib.sfe_remove_outlier_dev(ctx.handle, _dp(pts), _dp(off), n, int(pts.shape[1]), int(n_max),
                                              float(radius), int(min_points), _dp(out), _dp(idx), _dp(cnt)),
               "sfe_remove_outlier_dev")
    return dict(pts=out, idx=idx, count=cnt)


def match(ref_pts, ref_off, in_pts, in_off, n_ref_max, max_dist, knn=None, ctx=None):
    """Batched pcl.match (include/sonarfe.h: sfe_match_dev).  Without knn: the nearest reference point of every query,
    ids int32 and squared dists float32 [total query points].  With knn (1 .. 16, sfe_match_knn_dev): [knn, total]
    tensors whose row j holds every query's j-th nearest reference point within max_dist (-1 / +inf where there is
    none).  References of any size: those above one CTA's shared memory (whole maps) are searched as map grids in
    global memory, with the same results.  [total,3] points (both clouds): the 3-D distance (sfe_match_*_dim_dev)."""
    if knn is not None and int(knn) < 1:
        raise ValueError(f"ops.match: knn must be at least 1 (got {knn})")
    dim = int(ref_pts.shape[1])
    if dim not in (2, 3) or int(in_pts.shape[1]) != dim:
        raise ValueError(f"ops.match: reference and query points must both have 2 or 3 columns (got {dim} and "
                         f"{int(in_pts.shape[1])})")
    ctx = ctx or context(ref_pts.device)
    n = ref_off.numel() - 1
    shape = (in_pts.shape[0],) if knn is None else (int(knn), in_pts.shape[0])
    ids = torch.empty(shape, dtype=torch.int32, device=in_pts.device)
    d = torch.empty(shape, dtype=torch.float32, device=in_pts.device)
    if dim == 3:
        _lib.check(ctx.lib.sfe_match_knn_dim_dev(ctx.handle, _dp(ref_pts), _dp(ref_off), _dp(in_pts), _dp(in_off), n, 3,
                                                 int(n_ref_max), 1 if knn is None else int(knn), float(max_dist),
                                                 _dp(ids), _dp(d)), "sfe_match_knn_dim_dev")
    elif knn is None:
        _lib.check(ctx.lib.sfe_match_dev(ctx.handle, _dp(ref_pts), _dp(ref_off), _dp(in_pts), _dp(in_off), n,
                                         int(n_ref_max), float(max_dist), _dp(ids), _dp(d)), "sfe_match_dev")
    else:
        _lib.check(ctx.lib.sfe_match_knn_dev(ctx.handle, _dp(ref_pts), _dp(ref_off), _dp(in_pts), _dp(in_off), n,
                                             int(n_ref_max), int(knn), float(max_dist), _dp(ids), _dp(d)),
                   "sfe_match_knn_dev")
    return dict(ids=ids, dists=d)


def icp(src_pts, src_off, tgt_pts, tgt_off, guess, ns_max, nt_max, params=None, src_id=None, tgt_id=None, ctx=None,
        filters=None, robust=None):
    """Batched ICP (include/sonarfe.h: sfe_icp_dev).  guess: [P,3,3] f32 cuda.  Returns dict of cuda tensors.
    filters: _lib.IcpFilters (sfe_icp_set_filters), default params.filters when params is a parsed _lib.IcpConfig;
    its data filters (distance and octree) run on the device before the iterations.  robust: _lib.IcpRobust, the
    RobustOutlierFilter (sfe_icp_set_robust), default params.robust likewise; 2-D clouds only.

    Targets of any size: problems whose target does not fit one CTA's shared memory next to the sources read it from a
    map grid built once per distinct target (tgt_id) in global memory, with the same results.  Sources of any size:
    those above icp_source_limit (what the shared-memory layouts hold, about 8 400 points on an H100) take the
    global-source class -- their per-point arrays in global memory, every target read from a map grid -- with the same
    results.
    [total,3] points (both clouds) with [P,4,4] guesses: the 3-D point-to-point chain (sfe_icp_dim_dev), which takes no
    filters, robust filter, point-to-plane or float64 accumulation."""
    cols = [int(a.shape[1]) if a.dim() == 2 else 0 for a in (src_pts, tgt_pts)]
    dim = 3 if 3 in cols else 2
    if dim == 3 and cols != [3, 3]:
        raise ValueError(f"ops.icp: source and target points must have the same number of columns (got {cols})")
    if dim == 3 and (guess.dim() != 3 or tuple(guess.shape[1:]) != (4, 4)):
        raise ValueError(f"ops.icp: 3-column points take [P,4,4] guesses (got {list(guess.shape)})")
    ctx = ctx or context(src_pts.device)
    prm = params or _lib.IcpParams()
    guess = guess.contiguous()
    P = guess.shape[0]
    T = torch.empty((P, dim + 1, dim + 1), dtype=torch.float32, device=guess.device)
    iters = torch.empty((P,), dtype=torch.int32, device=guess.device)
    inl = torch.empty_like(iters)
    st = torch.empty_like(iters)
    _lib.set_icp_filters(ctx, _lib.icp_filters_of(prm, filters))
    _lib.set_icp_robust(ctx, _lib.icp_robust_of(prm, robust))
    if dim == 3:
        _lib.check(ctx.lib.sfe_icp_dim_dev(ctx.handle, ctypes.byref(prm), _dp(src_pts), _dp(src_off), _dp(tgt_pts),
                                           _dp(tgt_off), _dp(src_id), _dp(tgt_id), P, 3, int(ns_max), int(nt_max),
                                           _dp(guess), _dp(T), _dp(iters), _dp(inl), _dp(st)), "sfe_icp_dim_dev")
    else:
        _lib.check(ctx.lib.sfe_icp_dev(ctx.handle, ctypes.byref(prm), _dp(src_pts), _dp(src_off), _dp(tgt_pts),
                                       _dp(tgt_off), _dp(src_id), _dp(tgt_id), P, int(ns_max), int(nt_max), _dp(guess),
                                       _dp(T), _dp(iters), _dp(inl), _dp(st)), "sfe_icp_dev")
    return dict(T=T, iterations=iters, inliers=inl, status=st)


def icp_cta_limit(dim, ns, ctx=None, device=0):
    """The largest target of `dim` columns icp() solves in one CTA next to sources of ns points on this device
    (sfe_icp_cta_limit; dim 2: the shipped point-to-point chain without filters); larger targets take the map class."""
    ctx = ctx or context(device)
    out = np.zeros(1, np.int32)
    _lib.check(ctx.lib.sfe_icp_cta_limit(ctx.handle, int(dim), int(ns), _lib.ptr(out)), "sfe_icp_cta_limit")
    return int(out[0])


def icp_source_limit(dim, params=None, filters=None, ctx=None, device=0, robust=None):
    """The largest source of `dim` columns icp() solves in its shared-memory layouts next to targets of any size, for
    `params` (default _lib.IcpParams()), `filters` and `robust` (as icp() takes them) on this device
    (sfe_icp_source_limit).  Larger sources take the global-source class."""
    ctx = ctx or context(device)
    prm = params or _lib.IcpParams()
    _lib.set_icp_filters(ctx, _lib.icp_filters_of(prm, filters))
    _lib.set_icp_robust(ctx, _lib.icp_robust_of(prm, robust))
    out = np.zeros(1, np.int32)
    _lib.check(ctx.lib.sfe_icp_source_limit(ctx.handle, ctypes.byref(prm), int(dim), _lib.ptr(out)),
               "sfe_icp_source_limit")
    return int(out[0])


def surface_normals(pts, off, n_max, knn=5, ctx=None):
    """libpointmatcher's SurfaceNormalDataPointsFilter normals of packed 2-D clouds (include/sonarfe.h:
    sfe_icp_surface_normals_dev): pts [total,2] f32 cuda, off [n+1] int32 cuda (cloud c: rows off[c] .. off[c+1]),
    n_max >= every cloud's size (larger clouds are not read and their rows stay zero).  Returns [total,2] f32 cuda:
    every point's knn normal (3..16; ties to the lower index), in point order, computed on its cloud centred on the
    cloud's mean -- the reading normals of an ICP call with a SurfaceNormalDataPointsFilter in its reading chain."""
    ctx = ctx or context(pts.device)
    pts, off = pts.contiguous(), off.contiguous()
    out = torch.zeros_like(pts)
    _lib.check(ctx.lib.sfe_icp_surface_normals_dev(ctx.handle, _dp(pts), _dp(off), off.numel() - 1, int(n_max),
                                                   int(knn), _dp(out)), "sfe_icp_surface_normals_dev")
    return out


def mincovdet(samples, n, subsets, float32=False, ctx=None):
    """Batched MinCovDet(support_fraction=0.8) fits (include/sonarfe.h: sfe_mincovdet_dev; sonar_slam_b200/mcd.py).

    samples: float64 [P,32,3] cuda, n: int32 [P] cuda, subsets: int8 [P,30,32] cuda (mcd.draw_trial_supports).
    Returns dict(location=f64[P,3], covariance=f64[P,3,3], raw_support=i32[P], support=i32[P] (bit masks), status=i32[P]).
    """
    from . import mcd
    for name, t, dt in (("samples", samples, torch.float64), ("n", n, torch.int32), ("subsets", subsets, torch.int8)):
        if not t.is_cuda or t.dtype != dt:
            raise _lib.SonarFEError(f"ops.mincovdet: {name} must be a CUDA {dt} tensor")
    samples, n, subsets = samples.contiguous(), n.contiguous(), subsets.contiguous()
    P = n.numel()
    if samples.numel() != P * mcd.MAX_SAMPLES * 3 or subsets.numel() != P * mcd.TRIALS * mcd.MAX_SAMPLES:
        raise ValueError("ops.mincovdet: samples must be [P,32,3] and subsets [P,30,32]")
    ctx = ctx or context(samples.device)
    c, c_rw, cut = mcd.constants()
    dev = samples.device
    loc = torch.empty((P, 3), dtype=torch.float64, device=dev)
    cov = torch.empty((P, 3, 3), dtype=torch.float64, device=dev)
    raw = torch.empty((P,), dtype=torch.int32, device=dev)
    sup = torch.empty_like(raw)
    st = torch.empty_like(raw)
    _lib.check(ctx.lib.sfe_mincovdet_dev(ctx.handle, _dp(samples), _dp(n), _dp(subsets), P, _lib.ptr(c), c_rw, cut,
                                         mcd.FLOAT32 if float32 else 0, _dp(loc), _dp(cov), _dp(raw), _dp(sup), _dp(st)),
               "sfe_mincovdet_dev")
    return dict(location=loc, covariance=cov, raw_support=raw, support=sup, status=st)


def decode_jpeg(streams, R, B, device=None, ctx=None):
    """Decode compressed pings into a uint8 [n, R, B] tensor on the device (include/sonarfe.h: sfe_jpeg_decode_to_dev;
    sonar_slam_b200/jpeg.py).  streams: a sequence of bytes objects, or (bytes, offsets) from jpeg.pack.
    Returns (frames, status int32 [n] numpy): a frame whose status is not jpeg.OK is zeros.  The call returns once the
    frames are written (the statuses are read back)."""
    return _decode_to_dev("sfe_jpeg_decode_to_dev", streams, R, B, device, ctx)


def decode_png(streams, R, B, device=None, ctx=None):
    """decode_jpeg for PNG streams (include/sonarfe.h: sfe_png_decode_to_dev; sonar_slam_b200/png.py)."""
    return _decode_to_dev("sfe_png_decode_to_dev", streams, R, B, device, ctx)


def _decode_to_dev(name, streams, R, B, device, ctx):
    buf, off = _streams.packed(streams)
    n = len(off) - 1
    ctx = ctx or context(device)
    out = torch.empty((n, int(R), int(B)), dtype=torch.uint8, device=torch.device("cuda", ctx.device))
    st = np.empty(n, np.int32)
    _lib.check(getattr(ctx.lib, name)(ctx.handle, _lib.ptr(buf), _lib.ptr(off), n, int(R), int(B), _dp(out),
                                      _lib.ptr(st)), name)
    return out, st


def feature_image(frames, maps, lut=None, ctx=None):
    """Feature images (feature_extraction.py:226-228: cv2.remap + applyColorMap(JET)) of polar frames on the device
    (include/sonarfe.h: sfe_feature_image_dev; sonar_slam_b200/feature_image.py).  frames: uint8 [n, R, B] (or [R, B])
    cuda tensor of the maps' geometry; lut: uint8 [256, 3] BGR table (default feature_image.JET).
    Returns a uint8 [n, rows, cols, 3] bgr8 cuda tensor."""
    from . import feature_image as fimg
    if not frames.is_cuda or frames.dtype != torch.uint8:
        raise _lib.SonarFEError("ops.feature_image: frames must be a CUDA uint8 tensor")
    if frames.dim() == 2:
        frames = frames.unsqueeze(0)
    if frames.dim() != 3 or tuple(frames.shape[1:]) != (maps.R, maps.B):
        raise ValueError(f"ops.feature_image: frames must be [n, {maps.R}, {maps.B}] for these maps, "
                         f"got {tuple(frames.shape)}")
    frames = frames.contiguous()
    lut = fimg.lut_array(fimg.JET if lut is None else lut)
    ctx = ctx or context(frames.device)
    out = torch.empty((frames.shape[0], maps.rows, maps.cols, 3), dtype=torch.uint8, device=frames.device)
    _lib.check(ctx.lib.sfe_feature_image_dev(ctx.handle, maps.handle, _dp(frames), frames.shape[0], _lib.ptr(lut),
                                             _dp(out)), "sfe_feature_image_dev")
    return out
