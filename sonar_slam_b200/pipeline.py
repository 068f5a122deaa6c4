"""Batched per-keyframe front end (CFAR -> cloud -> filters -> sequential scan match).

Python face of include/sonarfe.h's sfe_frontend_*: one call per backlog of frames, inputs either
in host memory (`run_host`, the end-to-end path: frames are copied in chunks overlapped with the
kernels) or already on the device (`run_dev`).  See csrc/pipeline.cu for what is computed and how
it maps onto the reference's FeatureExtraction.callback / SLAM.add_sequential_scan_matching.
"""
import ctypes

import numpy as np

from . import _lib


class FrontEnd:
    def __init__(self, ctx, maps, max_frames, **overrides):
        """overrides: any field of sfe_frontend_params (e.g. tau=..., window=3, cap_points=4096) or
        `icp=_lib.IcpParams(...)`."""
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
        h = ctypes.c_void_p()
        _lib.check(self.lib.sfe_frontend_create(ctx.handle, maps.handle, ctypes.byref(p), self.max_frames,
                                                ctypes.byref(h)), "sfe_frontend_create")
        self.handle = h

    def run_host(self, frames, poses, chunk_frames=256, out=None):
        """frames: uint8 [n,R,B] numpy (pinned memory gives full copy bandwidth); poses: float64 [n,3].
        Returns dict(T [n,3,3] f32, iterations, inliers, status, npoints)."""
        frames = np.ascontiguousarray(frames, np.uint8)
        poses = np.ascontiguousarray(poses, np.float64)
        n = len(frames)
        o = out or self.alloc_results(n)
        _lib.check(self.lib.sfe_frontend_run_host(self.handle, _lib.ptr(frames), _lib.ptr(poses), n,
                                                  int(chunk_frames), _lib.ptr(o["T"]), _lib.ptr(o["iterations"]),
                                                  _lib.ptr(o["inliers"]), _lib.ptr(o["status"]),
                                                  _lib.ptr(o["npoints"])), "sfe_frontend_run_host")
        return o

    def run_jpeg_host(self, streams, poses, chunk_frames=256, out=None):
        """run_host on compressed pings: streams is a sequence of JPEG bytes objects (or (bytes, offsets) from
        jpeg.pack); the compressed bytes are copied and decoded on the device instead of copying raw frames
        (sfe_frontend_run_jpeg_host).  A stream that is rejected or fails to decode raises, naming the frame."""
        from . import jpeg
        buf, off = streams if isinstance(streams, tuple) else jpeg.pack(streams)
        poses = np.ascontiguousarray(poses, np.float64)
        n = len(off) - 1
        o = out or self.alloc_results(n)
        _lib.check(self.lib.sfe_frontend_run_jpeg_host(self.handle, _lib.ptr(buf), _lib.ptr(off), _lib.ptr(poses), n,
                                                       int(chunk_frames), _lib.ptr(o["T"]), _lib.ptr(o["iterations"]),
                                                       _lib.ptr(o["inliers"]), _lib.ptr(o["status"]),
                                                       _lib.ptr(o["npoints"])), "sfe_frontend_run_jpeg_host")
        return o

    def run_png_host(self, streams, poses, chunk_frames=256, out=None):
        """run_jpeg_host for PNG streams (sfe_frontend_run_png_host)."""
        from . import jpeg
        buf, off = streams if isinstance(streams, tuple) else jpeg.pack(streams)
        poses = np.ascontiguousarray(poses, np.float64)
        n = len(off) - 1
        o = out or self.alloc_results(n)
        _lib.check(self.lib.sfe_frontend_run_png_host(self.handle, _lib.ptr(buf), _lib.ptr(off), _lib.ptr(poses), n,
                                                      int(chunk_frames), _lib.ptr(o["T"]), _lib.ptr(o["iterations"]),
                                                      _lib.ptr(o["inliers"]), _lib.ptr(o["status"]),
                                                      _lib.ptr(o["npoints"])), "sfe_frontend_run_png_host")
        return o

    @staticmethod
    def alloc_results(n):
        return dict(T=np.empty((n, 3, 3), np.float32), iterations=np.empty(n, np.int32),
                    inliers=np.empty(n, np.int32), status=np.empty(n, np.int32), npoints=np.empty(n, np.int32))

    def run_dev(self, frames_ptr, poses, n):
        """frames_ptr: device address of uint8 [n,R,B]; poses: float64 [n,3] numpy (host).  Asynchronous."""
        poses = np.ascontiguousarray(poses, np.float64)
        _lib.check(self.lib.sfe_frontend_run_dev(self.handle, ctypes.c_void_p(int(frames_ptr)), _lib.ptr(poses),
                                                 int(n)), "sfe_frontend_run_dev")

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

    STAGES = ("cfar", "cart_points", "downsample", "remove_outlier", "submap", "icp")

    def set_timing(self, enable=True):
        _lib.check(self.lib.sfe_frontend_set_timing(self.handle, 1 if enable else 0), "sfe_frontend_set_timing")

    def get_timing(self):
        """dict stage -> (total ms, number of timed intervals) since set_timing(True)."""
        ms = np.zeros(len(self.STAGES), np.float64)
        calls = np.zeros(len(self.STAGES), np.int64)
        _lib.check(self.lib.sfe_frontend_get_timing(self.handle, _lib.ptr(ms), _lib.ptr(calls)), "sfe_frontend_get_timing")
        return {k: (float(ms[i]), int(calls[i])) for i, k in enumerate(self.STAGES)}

    def close(self):
        if getattr(self, "handle", None):
            self.lib.sfe_frontend_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
