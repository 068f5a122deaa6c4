"""PNG-compressed sonar pings decoded on the device (include/sonarfe.h: sfe_png_*; csrc/png.cu).

The reference decodes every ping of a compressed bag with cv2.imdecode(IMREAD_COLOR) + cvtColor(BGR2GRAY)
(feature_extraction.py:210-213).  For 8-bit gray or truecolour, non-interlaced PNG (any deflate content, any row
filter) the device decoder gives the same uint8 frames bit for bit; other streams (palette, alpha, 16-bit, Adam7,
APNG, JPEG ...) get a status naming the reason and stay on the host path.  The chunk list is walked on the host, so
`inspect` needs no GPU.  Streams are packed with jpeg.pack.
"""
import numpy as np

from . import _lib
from .jpeg import pack

(OK, NOT_PNG, TRUNCATED, BAD_HEADER, DEPTH, COLORTYPE, INTERLACED, ORIENTATION, ANIMATED, SIZE,
 CORRUPT) = range(11)                                     # SFE_PNG_* status
INFO_FIELDS = ("status", "height", "width", "colour_type", "idat_chunks")
SIGNATURE = b"\x89PNG\r\n\x1a\n"


def status_message(status):
    return _lib.load().sfe_png_status_message(int(status)).decode()


def inspect(streams):
    """Chunk list only (no GPU): int32 [n, 5] rows (status, height, width, colour type, IDAT chunks)."""
    buf, off = streams if isinstance(streams, tuple) else pack(streams)
    n = len(off) - 1
    info = np.zeros((n, len(INFO_FIELDS)), np.int32)
    _lib.check(_lib.load().sfe_png_inspect_host(_lib.ptr(buf), _lib.ptr(off), n, _lib.ptr(info)),
               "sfe_png_inspect_host")
    return info


def decode_host(streams, R, B, ctx=None):
    """Decode into host memory: (uint8 [n, R, B], status int32 [n]); a frame whose status is not OK is zeros."""
    ctx = ctx or _lib.default_context()
    buf, off = streams if isinstance(streams, tuple) else pack(streams)
    n = len(off) - 1
    out = np.zeros((n, int(R), int(B)), np.uint8)
    st = np.zeros(n, np.int32)
    _lib.check(ctx.lib.sfe_png_decode_host(ctx.handle, _lib.ptr(buf), _lib.ptr(off), n, int(R), int(B),
                                           _lib.ptr(out), _lib.ptr(st)), "sfe_png_decode_host")
    return out, st


STAGES = ("check", "inflate", "unfilter")


def set_timing(enable=True, ctx=None):
    """Per-stage device timing of the decoder on this context (CUDA events around every chunk's kernels)."""
    ctx = ctx or _lib.default_context()
    _lib.check(ctx.lib.sfe_png_set_timing(ctx.handle, 1 if enable else 0), "sfe_png_set_timing")


def get_timing(ctx=None):
    """dict stage -> (total ms, number of timed intervals) since set_timing(True)."""
    ctx = ctx or _lib.default_context()
    ms = np.zeros(len(STAGES), np.float64)
    calls = np.zeros(len(STAGES), np.int64)
    _lib.check(ctx.lib.sfe_png_get_timing(ctx.handle, _lib.ptr(ms), _lib.ptr(calls)), "sfe_png_get_timing")
    return {k: (float(ms[i]), int(calls[i])) for i, k in enumerate(STAGES)}
