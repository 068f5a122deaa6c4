"""Batched per-keyframe front end (CFAR -> cloud -> filters -> sequential scan match).

Python face of include/sonarfe.h's sfe_frontend_*: one call per backlog of frames, inputs either
in host memory (`run_host`, the end-to-end path: frames are copied in chunks overlapped with the
kernels) or already on the device (`run_dev`).  See csrc/pipeline.cu for what is computed and how
it maps onto the reference's FeatureExtraction.callback / SLAM.add_sequential_scan_matching.
"""
import contextlib
import ctypes

import numpy as np

from . import _lib, _streams


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

    @contextlib.contextmanager
    def _images(self, images, n, on_device, lut):
        """Feature images of the frames of one run call (sfe_frontend_set_feature_images), off again afterwards.
        images: uint8 [n, rows, cols, 3] C-contiguous -- a numpy array for the host flavours, a CUDA tensor on the
        context's device for run_dev; lut: uint8 [256, 3] BGR table (default feature_image.JET)."""
        if images is None:
            yield
            return
        from . import feature_image
        shape = (n, self.maps.rows, self.maps.cols, 3)
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

    def run_host(self, frames, poses, chunk_frames=256, out=None, images=None, image_lut=None):
        """frames: uint8 [n,R,B] numpy (pinned memory gives full copy bandwidth); poses: float64 [n,3].
        Returns dict(T [n,3,3] f32, iterations, inliers, status, npoints).  images: an optional uint8
        [n, rows, cols, 3] numpy array that receives every frame's feature image (feature_image.py; colour table
        image_lut, default JET); the results are the same with and without it."""
        frames = np.ascontiguousarray(frames, np.uint8)
        poses = np.ascontiguousarray(poses, np.float64)
        n = len(frames)
        o = out or self.alloc_results(n)
        with self._images(images, n, False, image_lut):
            _lib.check(self.lib.sfe_frontend_run_host(self.handle, _lib.ptr(frames), _lib.ptr(poses), n,
                                                      int(chunk_frames), _lib.ptr(o["T"]), _lib.ptr(o["iterations"]),
                                                      _lib.ptr(o["inliers"]), _lib.ptr(o["status"]),
                                                      _lib.ptr(o["npoints"])), "sfe_frontend_run_host")
        return o

    def run_jpeg_host(self, streams, poses, chunk_frames=256, out=None, images=None, image_lut=None):
        """run_host on compressed pings: streams is a sequence of JPEG bytes objects (or (bytes, offsets) from
        jpeg.pack); the compressed bytes are copied and decoded on the device instead of copying raw frames
        (sfe_frontend_run_jpeg_host).  A stream that is rejected or fails to decode raises, naming the frame.
        images / image_lut: as run_host."""
        return self._run_compressed("sfe_frontend_run_jpeg_host", streams, poses, chunk_frames, out, images, image_lut)

    def run_png_host(self, streams, poses, chunk_frames=256, out=None, images=None, image_lut=None):
        """run_jpeg_host for PNG streams (sfe_frontend_run_png_host)."""
        return self._run_compressed("sfe_frontend_run_png_host", streams, poses, chunk_frames, out, images, image_lut)

    def _run_compressed(self, name, streams, poses, chunk_frames, out, images, image_lut):
        buf, off = _streams.packed(streams)
        poses = np.ascontiguousarray(poses, np.float64)
        n = len(off) - 1
        o = out or self.alloc_results(n)
        with self._images(images, n, False, image_lut):
            _lib.check(getattr(self.lib, name)(self.handle, _lib.ptr(buf), _lib.ptr(off), _lib.ptr(poses), n,
                                               int(chunk_frames), _lib.ptr(o["T"]), _lib.ptr(o["iterations"]),
                                               _lib.ptr(o["inliers"]), _lib.ptr(o["status"]), _lib.ptr(o["npoints"])),
                       name)
        return o

    @staticmethod
    def alloc_results(n):
        return dict(T=np.empty((n, 3, 3), np.float32), iterations=np.empty(n, np.int32),
                    inliers=np.empty(n, np.int32), status=np.empty(n, np.int32), npoints=np.empty(n, np.int32))

    def run_dev(self, frames_ptr, poses, n, images=None, image_lut=None):
        """frames_ptr: device address of uint8 [n,R,B]; poses: float64 [n,3] numpy (host).  Asynchronous.
        images: an optional uint8 [n, rows, cols, 3] CUDA tensor that receives every frame's feature image."""
        poses = np.ascontiguousarray(poses, np.float64)
        with self._images(images, int(n), True, image_lut):
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

    def set_overlap(self, sub_batch_frames):
        """Schedule of run_dev (sfe_frontend_set_overlap): > 0 overlaps the feature stages of one sub-batch of that
        many frames with the scan matching of the previous one on two streams; 0 (the default) runs every stage over
        the whole batch one after another.  The results are the same either way."""
        _lib.check(self.lib.sfe_frontend_set_overlap(self.handle, int(sub_batch_frames)), "sfe_frontend_set_overlap")

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
