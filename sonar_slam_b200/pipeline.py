"""Batched per-keyframe front end (CFAR -> cloud -> filters -> sequential scan match).

Python face of include/sonarfe.h's sfe_frontend_*: one call per backlog of frames, inputs either
in host memory (`run_host`, the end-to-end path: frames are copied in chunks overlapped with the
kernels) or already on the device (`run_dev`).  See csrc/pipeline.cu for what is computed and how
it maps onto the reference's FeatureExtraction.callback / SLAM.add_sequential_scan_matching.

A front end may hold several sonar geometries (add_geometry): every run flavour then takes `geometry=`, one id per
frame, and a bag whose range setting changes is fed as one sequence.
"""
import contextlib
import ctypes

import numpy as np

from . import _lib, _streams


class FrontEnd:
    def __init__(self, ctx, maps, max_frames, icp_filters=None, icp_robust=None, **overrides):
        """overrides: any field of sfe_frontend_params (e.g. tau=..., window=3, cap_points=4096) or
        `icp=_lib.IcpParams(...)`.  icp_filters: _lib.IcpFilters of the scan match (sfe_frontend_set_icp_filters),
        default icp.filters when `icp` is a parsed _lib.IcpConfig; icp_robust: its _lib.IcpRobust
        (sfe_frontend_set_icp_robust), default icp.robust likewise."""
        self.ctx, self.maps, self.lib = ctx, maps, ctx.lib
        p = _lib.FrontendParams()
        self.lib.sfe_frontend_params_default(ctypes.byref(p))
        p.R, p.B = maps.R, maps.B
        for k, v in overrides.items():
            if not hasattr(p, k):
                raise TypeError(f"unknown front-end parameter {k!r}")
            setattr(p, k, v)
        self.params = p
        self.max_frames = int(max_frames)
        self.geometries = [maps]  # id -> Maps (kept alive: the front end references them)
        h = ctypes.c_void_p()
        _lib.check(self.lib.sfe_frontend_create(ctx.handle, maps.handle, ctypes.byref(p), self.max_frames,
                                                ctypes.byref(h)), "sfe_frontend_create")
        self.handle = h
        filters = _lib.icp_filters_of(overrides.get("icp"), icp_filters)
        if filters is not None:
            _lib.check(self.lib.sfe_frontend_set_icp_filters(h, ctypes.byref(filters)), "sfe_frontend_set_icp_filters")
        robust = _lib.icp_robust_of(overrides.get("icp"), icp_robust)
        if robust is not None:
            _lib.check(self.lib.sfe_frontend_set_icp_robust(h, ctypes.byref(robust)), "sfe_frontend_set_icp_robust")

    def add_geometry(self, maps):
        """Register a further sonar geometry (sfe_frontend_add_geometry) and return its id; the creation maps are
        geometry 0.  Its polar shape must fit the frame slots the front end was created with (maps.R <= R,
        maps.B <= B); at most _lib.MAX_GEOMETRIES geometries."""
        gid = ctypes.c_int()
        _lib.check(self.lib.sfe_frontend_add_geometry(self.handle, maps.handle, ctypes.byref(gid)),
                   "sfe_frontend_add_geometry")
        self.geometries.append(maps)
        return gid.value

    def _geometry(self, geometry, n):
        """geometry= of a run call -> int32 [n] (or None)."""
        if geometry is None:
            return None
        g = np.ascontiguousarray(geometry, np.int32).reshape(-1)
        if len(g) != n:
            raise ValueError(f"FrontEnd: geometry has {len(g)} ids for {n} frames")
        return g

    def _image_maps(self, geometry):
        """The geometry whose feature images a call writes: its frames' one geometry (several: the C side refuses)."""
        if geometry is None or len(geometry) == 0 or not 0 <= geometry[0] < len(self.geometries):
            return self.maps
        return self.geometries[geometry[0]]

    def pack_frames(self, frames, geometry):
        """Raw frames of several geometries -> (uint8 bytes [total], int64 offsets [n + 1]), frame i =
        bytes[offsets[i]:offsets[i + 1]] row-major [R_g, B_g] (the host form of sfe_frontend_run_host_geometry).
        frames: a sequence of uint8 [R_g, B_g] arrays, or (bytes, offsets) already packed, which is checked."""
        if isinstance(frames, tuple):
            buf, off = frames
            buf = np.ascontiguousarray(buf, np.uint8).reshape(-1)
            off = np.ascontiguousarray(off, np.int64)
            if off.ndim != 1 or len(off) == 0 or off[0] < 0 or off[-1] > buf.size:
                raise ValueError(f"FrontEnd: frame offsets overrun the packed buffer ({buf.size} bytes)")
            return buf, off
        for i, f in enumerate(frames):
            g = int(geometry[i]) if i < len(geometry) else 0
            if 0 <= g < len(self.geometries):
                m = self.geometries[g]
                if np.shape(f) != (m.R, m.B):
                    raise ValueError(f"FrontEnd: frame {i} has shape {np.shape(f)}; its geometry {g} is "
                                     f"{m.R} x {m.B}")
        return _streams.pack(np.ascontiguousarray(f, np.uint8).tobytes() for f in frames)

    @contextlib.contextmanager
    def _images(self, images, n, on_device, lut, maps=None):
        """Feature images of the frames of one run call (sfe_frontend_set_feature_images), off again afterwards.
        images: uint8 [n, rows, cols, 3] C-contiguous -- a numpy array for the host flavours, a CUDA tensor on the
        context's device for run_dev; lut: uint8 [256, 3] BGR table (default feature_image.JET)."""
        if images is None:
            yield
            return
        from . import feature_image
        maps = maps or self.maps
        shape = (n, maps.rows, maps.cols, 3)
        if on_device:
            import torch
            if not (isinstance(images, torch.Tensor) and images.is_cuda and images.dtype == torch.uint8
                    and tuple(images.shape) == shape and images.is_contiguous()):
                raise ValueError(f"FrontEnd.run_dev: images must be a contiguous CUDA uint8 tensor {list(shape)}")
            dst = images.data_ptr()
        else:
            if not (isinstance(images, np.ndarray) and images.dtype == np.uint8 and images.shape == shape
                    and images.flags["C_CONTIGUOUS"] and images.flags["WRITEABLE"]):
                raise ValueError(f"FrontEnd: images must be a writeable C-contiguous uint8 numpy array {list(shape)}")
            dst = images.ctypes.data
        lut = feature_image.lut_array(feature_image.JET if lut is None else lut)
        _lib.check(self.lib.sfe_frontend_set_feature_images(self.handle, _lib.ptr(lut), ctypes.c_void_p(dst),
                                                            0 if on_device else 1), "sfe_frontend_set_feature_images")
        try:
            yield
        finally:
            self.lib.sfe_frontend_set_feature_images(self.handle, None, None, 0)

    def _with_clouds(self, clouds, n, on_device, name, call):
        """Run `call()` (one run call, returning its status code) with packed clouds when `clouds` asks for them
        (sfe_frontend_set_clouds), off again afterwards; returns None or (points float32 [total, 2], offsets int64
        [n + 1]) -- numpy arrays for the host flavours, CUDA tensors on the context's device for run_dev.
        clouds: None / False (none), True (a buffer of the bound n * cap_points: every frame's cloud has at most
        cap_points points; a numpy buffer only commits the pages written), an int (that capacity in points; a call whose
        clouds need more is run once more with a buffer of the total it reports -- it left the carried window as it
        was), or, for run_dev, (points, offsets) CUDA tensors of the caller, float32 [capacity, 2] and int64 [n + 1]
        contiguous, which are filled (a call that overflows them raises)."""
        if clouds is None or clouds is False:
            _lib.check(call(), name)
            return None
        own = not isinstance(clouds, tuple)
        if own:
            cap = n * self.params.cap_points if clouds is True else int(clouds)
            if cap < 0:
                raise ValueError(f"FrontEnd: clouds capacity {cap} is negative")
        else:
            if not on_device:
                raise ValueError("FrontEnd: caller-provided cloud buffers are for run_dev; the host flavours take "
                                 "clouds=True or a capacity")
            import torch
            pts, off = clouds
            for t, dt, shape in ((pts, torch.float32, None), (off, torch.int64, (n + 1,))):
                if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dt and t.is_contiguous()
                        and (t.shape == shape if shape else (t.dim() == 2 and t.shape[1] == 2))):
                    raise ValueError("FrontEnd.run_dev: clouds must be contiguous CUDA tensors float32 [capacity, 2] "
                                     f"and int64 [{n + 1}]")
            cap = pts.shape[0]
        for attempt in (0, 1):
            if own and on_device:
                import torch
                dev = torch.device("cuda", self.ctx.device)
                pts = torch.empty((max(cap, 1), 2), dtype=torch.float32, device=dev)
                off = torch.empty(n + 1, dtype=torch.int64, device=dev)
            elif own:
                pts, off = np.empty((max(cap, 1), 2), np.float32), np.zeros(n + 1, np.int64)
            if on_device:
                dst, offsets = ctypes.c_void_p(pts.data_ptr()), ctypes.c_void_p(off.data_ptr())
            else:
                dst, offsets = _lib.ptr(pts), _lib.ptr(off)
            _lib.check(self.lib.sfe_frontend_set_clouds(self.handle, dst, cap, offsets, 0 if on_device else 1),
                       "sfe_frontend_set_clouds")
            try:
                rc = call()
            finally:
                self.lib.sfe_frontend_set_clouds(self.handle, None, 0, None, 0)
            if rc == _lib.ERR_CAPACITY and own and attempt == 0 and clouds is not True:
                cap = int(off[-1])
                continue
            _lib.check(rc, name)
            return pts[:int(off[-1])], off

    def run_host(self, frames, poses, chunk_frames=256, out=None, images=None, image_lut=None, geometry=None,
                 clouds=None):
        """frames: uint8 [n,R,B] numpy (pinned memory gives full copy bandwidth); poses: float64 [n,3].
        Returns dict(T [n,3,3] f32, iterations, inliers, status, npoints).  images: an optional uint8
        [n, rows, cols, 3] numpy array that receives every frame's feature image (feature_image.py; colour table
        image_lut, default JET); the results are the same with and without it.
        geometry: one id per frame (add_geometry); frames are then a sequence of uint8 [R_g, B_g] arrays or
        (bytes, offsets) from pack_frames (sfe_frontend_run_host_geometry).
        clouds: True or a capacity in points (see _with_clouds) adds every frame's filtered cloud, packed: "clouds"
        float32 [total, 2] and "cloud_offsets" int64 [n + 1], frame i = clouds[cloud_offsets[i]:cloud_offsets[i + 1]]
        in the flip_lateral convention; the other results are the same with and without them."""
        if geometry is None:
            frames = np.ascontiguousarray(frames, np.uint8)
            n = len(frames)
            head = (_lib.ptr(frames),)
        else:
            n = len(frames[1]) - 1 if isinstance(frames, tuple) else len(frames)
            geometry = self._geometry(geometry, n)
            buf, off = self.pack_frames(frames, geometry)
            head = (_lib.ptr(buf), _lib.ptr(off))
        return self._run_host("sfe_frontend_run_host", head, poses, n, chunk_frames, out, images, image_lut, geometry,
                              clouds)

    def run_jpeg_host(self, streams, poses, chunk_frames=256, out=None, images=None, image_lut=None, geometry=None,
                      clouds=None):
        """run_host on compressed pings: streams is a sequence of JPEG bytes objects (or (bytes, offsets) from
        jpeg.pack); the compressed bytes are copied and decoded on the device instead of copying raw frames
        (sfe_frontend_run_jpeg_host).  A stream that is rejected or fails to decode raises, naming the frame.
        images / image_lut / geometry / clouds: as run_host (with geometry, every stream must decode to its geometry's
        R_g x B_g)."""
        return self._run_compressed("sfe_frontend_run_jpeg_host", streams, poses, chunk_frames, out, images, image_lut,
                                    geometry, clouds)

    def run_png_host(self, streams, poses, chunk_frames=256, out=None, images=None, image_lut=None, geometry=None,
                     clouds=None):
        """run_jpeg_host for PNG streams (sfe_frontend_run_png_host)."""
        return self._run_compressed("sfe_frontend_run_png_host", streams, poses, chunk_frames, out, images, image_lut,
                                    geometry, clouds)

    def _run_compressed(self, name, streams, poses, chunk_frames, out, images, image_lut, geometry, clouds):
        buf, off = _streams.packed(streams)
        n = len(off) - 1
        return self._run_host(name, (_lib.ptr(buf), _lib.ptr(off)), poses, n, chunk_frames, out, images, image_lut,
                              self._geometry(geometry, n), clouds)

    def _run_host(self, name, head, poses, n, chunk_frames, out, images, image_lut, geometry, clouds):
        """A host flavour's call (see _run) into `out` or new result arrays, with the packed clouds added."""
        o = out or self.alloc_results(n)
        tail = (int(chunk_frames),) + tuple(_lib.ptr(o[k]) for k in ("T", "iterations", "inliers", "status", "npoints"))
        packed = self._run(name, head, poses, n, geometry, False, images, image_lut, clouds, tail)
        if packed is not None:
            o["clouds"], o["cloud_offsets"] = packed
        return o

    def _run(self, name, head, poses, n, geometry, on_device, images, image_lut, clouds, tail=()):
        """One run call: entry point `name` (its _geometry form when geometry is given) with the leading arguments
        `head`, then the geometry, poses, n and `tail`; the call's feature images and packed clouds around it (the
        latter returned, see _with_clouds)."""
        poses = np.ascontiguousarray(poses, np.float64)
        head = (self.handle,) + head
        if geometry is not None:
            name, head = name + "_geometry", head + (_lib.ptr(geometry),)
        with self._images(images, n, on_device, image_lut, self._image_maps(geometry)):
            return self._with_clouds(clouds, n, on_device, name,
                                     lambda: getattr(self.lib, name)(*head, _lib.ptr(poses), n, *tail))

    @staticmethod
    def alloc_results(n):
        return dict(T=np.empty((n, 3, 3), np.float32), iterations=np.empty(n, np.int32),
                    inliers=np.empty(n, np.int32), status=np.empty(n, np.int32), npoints=np.empty(n, np.int32))

    def run_dev(self, frames_ptr, poses, n, images=None, image_lut=None, geometry=None, clouds=None):
        """frames_ptr: device address of uint8 [n,R,B]; poses: float64 [n,3] numpy (host).  Asynchronous.
        images: an optional uint8 [n, rows, cols, 3] CUDA tensor that receives every frame's feature image.
        geometry: one id per frame (add_geometry); frame i of geometry g then occupies the first R_g * B_g bytes of
        its R * B slot, row-major [R_g, B_g] (sfe_frontend_run_dev_geometry).
        clouds: True, a capacity or (points, offsets) CUDA tensors (see _with_clouds): every frame's filtered cloud,
        packed on the device, and the call returns (points [total, 2], offsets [n + 1]) CUDA tensors once the call has
        finished; without clouds it returns None."""
        n = int(n)
        return self._run("sfe_frontend_run_dev", (ctypes.c_void_p(int(frames_ptr)),), poses, n,
                         self._geometry(geometry, n), True, images, image_lut, clouds)

    def results_dev(self):
        """Device addresses of the last run's results: dict(T, iterations, inliers, status, cloud_xy,
        cloud_count, cloud_stride)."""
        ptrs = [ctypes.c_void_p() for _ in range(6)]
        stride = ctypes.c_int32()
        _lib.check(self.lib.sfe_frontend_results_dev(self.handle, *[ctypes.byref(q) for q in ptrs],
                                                     ctypes.byref(stride)), "sfe_frontend_results_dev")
        names = ["T", "iterations", "inliers", "status", "cloud_xy", "cloud_count"]
        d = {k: q.value for k, q in zip(names, ptrs)}
        d["cloud_stride"] = stride.value
        return d

    def set_carry(self, enable=True):
        """Continue the frame sequence across calls: the last `window` clouds and poses stay on the device and serve
        as the window of the next call's first frames (sfe_frontend_set_carry).  False: every call starts cold."""
        _lib.check(self.lib.sfe_frontend_set_carry(self.handle, 1 if enable else 0), "sfe_frontend_set_carry")

    def set_scan_match(self, enable=True):
        """False: every run flavour stops after the feature stages (sfe_frontend_set_scan_match): no window submaps,
        no ICP; status SKIPPED (TOO_LARGE where a Cartesian cloud overflowed cap_points), T the identity.  The clouds
        are the same either way; with carry on the carried window still advances."""
        _lib.check(self.lib.sfe_frontend_set_scan_match(self.handle, 1 if enable else 0), "sfe_frontend_set_scan_match")

    STAGES = ("cfar", "cart_points", "downsample", "remove_outlier", "submap", "icp")

    def set_timing(self, enable=True):
        _lib.check(self.lib.sfe_frontend_set_timing(self.handle, 1 if enable else 0), "sfe_frontend_set_timing")

    def get_timing(self):
        """dict stage -> (total ms, number of timed intervals) since set_timing(True)."""
        return _streams.read_timing(self.lib.sfe_frontend_get_timing, self.handle, self.STAGES)

    def close(self):
        if getattr(self, "handle", None):
            self.lib.sfe_frontend_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
