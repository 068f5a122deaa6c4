"""Bodies shared by the compressed-stream decoders (jpeg.py, png.py) and the stage timers (pipeline.FrontEnd).

A codec's entry points are named sfe_<codec>_<what> (include/sonarfe.h); `prefix` is the sfe_<codec>_ part.
"""
import numpy as np

from . import _lib


def pack(streams):
    """Sequence of byte strings -> (uint8 bytes [total], int64 offsets [n + 1])."""
    streams = [bytes(s) for s in streams]
    off = np.zeros(len(streams) + 1, np.int64)
    off[1:] = np.cumsum([len(s) for s in streams])
    buf = np.frombuffer(b"".join(streams), np.uint8) if off[-1] else np.zeros(1, np.uint8)
    return np.ascontiguousarray(buf), off


def packed(streams):
    """(bytes, offsets) as given, or pack(streams)."""
    return streams if isinstance(streams, tuple) else pack(streams)


def inspect(prefix, streams, fields):
    buf, off = packed(streams)
    n = len(off) - 1
    info = np.zeros((n, len(fields)), np.int32)
    name = prefix + "inspect_host"
    _lib.check(getattr(_lib.load(), name)(_lib.ptr(buf), _lib.ptr(off), n, _lib.ptr(info)), name)
    return info


def decode_host(prefix, streams, R, B, ctx):
    ctx = ctx or _lib.default_context()
    buf, off = packed(streams)
    n = len(off) - 1
    out = np.zeros((n, int(R), int(B)), np.uint8)
    st = np.zeros(n, np.int32)
    name = prefix + "decode_host"
    _lib.check(getattr(ctx.lib, name)(ctx.handle, _lib.ptr(buf), _lib.ptr(off), n, int(R), int(B), _lib.ptr(out),
                                      _lib.ptr(st)), name)
    return out, st


def set_timing(prefix, enable, ctx):
    ctx = ctx or _lib.default_context()
    name = prefix + "set_timing"
    _lib.check(getattr(ctx.lib, name)(ctx.handle, 1 if enable else 0), name)


def get_timing(prefix, stages, ctx):
    ctx = ctx or _lib.default_context()
    return read_timing(getattr(ctx.lib, prefix + "get_timing"), ctx.handle, stages)


def read_timing(fn, handle, stages):
    """dict stage -> (total ms, number of timed intervals) from one of the sfe_*_get_timing entry points."""
    ms = np.zeros(len(stages), np.float64)
    calls = np.zeros(len(stages), np.int64)
    _lib.check(fn(handle, _lib.ptr(ms), _lib.ptr(calls)), fn.__name__)
    return {k: (float(ms[i]), int(calls[i])) for i, k in enumerate(stages)}
