"""Keyframe clouds resident on the device (include/sonarfe.h: sfe_keyframe_map_*).

SLAM.get_points (slam.py:229-292) moves every selected keyframe's cloud into one frame, concatenates and down-samples.
A `KeyframeMap` stores each cloud once, in its local coordinates, and assembles any selection under new poses on the
device, with pcl.downsample's results: only the entries (slot, key, 6-float transform) go to the device per call.
bruce_slam.slam.SLAM() keeps its keyframes in a list backed by one of these (bruce_slam.slam.KeyframeList).
"""
import ctypes

import numpy as np

from . import _lib


def _addr(x):
    """Device address of a torch tensor or a raw address (int)."""
    return x.data_ptr() if hasattr(x, "data_ptr") else int(x)


class KeyframeMap:
    """One device arena of keyframe clouds owned by one context (sfe_keyframe_map); not thread-safe."""

    def __init__(self, ctx=None, capacity=0):
        """capacity: points the arena holds before it first grows (0: the library's default)."""
        self.ctx = ctx or _lib.default_context()
        self.lib = self.ctx.lib
        h = ctypes.c_void_p()
        _lib.check(self.lib.sfe_keyframe_map_create(self.ctx.handle, int(capacity), ctypes.byref(h)),
                   "sfe_keyframe_map_create")
        self.handle = h
        self.counts = np.zeros(0, np.int64)  # points of every slot

    def append(self, points):
        """Store the clouds of `points` (a sequence of float32-convertible [N, 2] arrays) in one upload; returns their
        slot ids (int32)."""
        clouds = [np.ascontiguousarray(p, np.float32) for p in points]
        for c in clouds:
            if c.ndim != 2 or c.shape[1] != 2:
                raise ValueError(f"KeyframeMap.append: clouds must be [N, 2], got {c.shape}")
        counts = np.array([len(c) for c in clouds], np.int32)
        packed = np.ascontiguousarray(np.concatenate(clouds + [np.zeros((0, 2), np.float32)]))
        slots = np.empty(len(clouds), np.int32)
        _lib.check(self.lib.sfe_keyframe_map_append_host(self.handle, _lib.ptr(packed), _lib.ptr(counts), len(clouds),
                                                         _lib.ptr(slots)), "sfe_keyframe_map_append_host")
        self.counts = np.r_[self.counts, counts]
        return slots

    def append_dev(self, xy, count, stride, n):
        """Store n clouds already on the device in FrontEnd.results_dev()'s layout (cloud c: count[c] points at
        xy + 2 * c * stride floats; xy and count are device addresses or torch tensors); returns their slot ids."""
        slots = np.empty(int(n), np.int32)
        counts = np.empty(int(n), np.int32)
        _lib.check(self.lib.sfe_keyframe_map_append_dev(self.handle, ctypes.c_void_p(_addr(xy)),
                                                        ctypes.c_void_p(_addr(count)), int(stride), int(n),
                                                        _lib.ptr(slots), _lib.ptr(counts)),
                   "sfe_keyframe_map_append_dev")
        self.counts = np.r_[self.counts, counts]
        return slots

    @property
    def size(self):
        """(clouds, points) stored."""
        n, p = ctypes.c_int(), ctypes.c_int64()
        _lib.check(self.lib.sfe_keyframe_map_size(self.handle, ctypes.byref(n), ctypes.byref(p)), "sfe_keyframe_map_size")
        return n.value, p.value

    def assemble(self, slots, keys, transforms, resolution, with_keys, device=False):
        """The clouds of `slots` (int [K], repeats allowed), entry k moved by transforms[k] = {r00, r01, r10, r11, tx,
        ty} (float32 [K, 6]) and carrying keys[k] (float32 [K]; may be None without keys), concatenated in entry order
        and down-sampled at `resolution`.  Returns points float32 [M, 2], or (points, keys float32 [M]) with_keys:
        numpy arrays, or with device=True torch tensors on the context's device (the call returns once M is known)."""
        slots = np.ascontiguousarray(slots, np.int32).reshape(-1)
        K = len(slots)
        tf = np.ascontiguousarray(transforms, np.float32).reshape(K, 6)
        kk = np.ascontiguousarray(keys, np.float32).reshape(K) if with_keys else None
        bad = (slots < 0) | (slots >= len(self.counts))
        if bad.any():
            raise IndexError(f"KeyframeMap.assemble: slot {int(slots[bad][0])} is not stored "
                             f"({len(self.counts)} clouds)")
        n = int(self.counts[slots].sum())
        if device:
            return self._assemble_dev(slots, kk, tf, resolution, with_keys, n)
        pts = np.empty((n, 2), np.float32)
        out_keys = np.empty(n, np.float32) if with_keys else None
        m = np.zeros(1, np.int32)
        _lib.check(self.lib.sfe_keyframe_map_assemble_host(self.handle, _lib.ptr(slots), _lib.ptr(kk), _lib.ptr(tf), K,
                                                           float(resolution), n, _lib.ptr(pts), _lib.ptr(out_keys),
                                                           _lib.ptr(m)), "sfe_keyframe_map_assemble_host")
        k = int(m[0])
        return (pts[:k], out_keys[:k]) if with_keys else pts[:k]

    def _assemble_dev(self, slots, kk, tf, resolution, with_keys, n):
        import torch
        dev = torch.device("cuda", self.ctx.device)
        pts = torch.empty((n, 2), dtype=torch.float32, device=dev)
        out_keys = torch.empty((n,), dtype=torch.float32, device=dev) if with_keys else None
        m = torch.zeros((1,), dtype=torch.int32, device=dev)
        # the outputs come from torch's allocator on its current stream, the work runs on the context's: let torch's
        # earlier work on those blocks finish first
        torch.cuda.current_stream(dev).synchronize()
        _lib.check(self.lib.sfe_keyframe_map_assemble_dev(self.handle, _lib.ptr(slots), _lib.ptr(kk), _lib.ptr(tf),
                                                          len(slots), float(resolution), n,
                                                          ctypes.c_void_p(pts.data_ptr()),
                                                          ctypes.c_void_p(out_keys.data_ptr()) if with_keys else None,
                                                          ctypes.c_void_p(m.data_ptr())),
                   "sfe_keyframe_map_assemble_dev")
        k = int(self.ctx.to_host(m.data_ptr(), (1,), np.int32)[0])  # synchronises the context's stream
        return (pts[:k], out_keys[:k]) if with_keys else pts[:k]

    def close(self):
        if getattr(self, "handle", None):
            self.lib.sfe_keyframe_map_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
