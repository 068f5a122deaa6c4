"""Compressed sonar pings decoded on the device (include/sonarfe.h: sfe_jpeg_*; csrc/jpeg.cu).

The reference decodes every ping of a compressed bag with cv2.imdecode(IMREAD_COLOR) + cvtColor(BGR2GRAY)
(feature_extraction.py:210-213).  For baseline / extended sequential JPEG (gray, or YCbCr at 4:4:4, 4:2:2, 4:2:0, any
restart interval) the device decoder gives the same uint8 frames bit for bit; other streams (progressive, PNG, ...) get a
status naming the reason and stay on the host path.  Headers are parsed on the host, so `inspect` needs no GPU.
"""
import numpy as np

from . import _lib, _streams
from ._streams import pack  # noqa: F401  (jpeg.pack: the packing of every codec)

(OK, NOT_JPEG, TRUNCATED, PROGRESSIVE, LOSSLESS, ARITHMETIC, PRECISION, SAMPLING, COLORSPACE, ORIENTATION, SIZE,
 CORRUPT, BAD_HEADER) = range(13)                         # SFE_JPEG_* status
GRAY, S444, S422, S420 = range(4)                        # sampling codes
INFO_FIELDS = ("status", "height", "width", "components", "sampling", "restart_interval")


def status_message(status):
    return _lib.load().sfe_jpeg_status_message(int(status)).decode()


def inspect(streams):
    """Headers only (no GPU): int32 [n, 6] rows (status, height, width, components, sampling, restart interval)."""
    return _streams.inspect("sfe_jpeg_", streams, INFO_FIELDS)


def decode_host(streams, R, B, ctx=None):
    """Decode into host memory: (uint8 [n, R, B], status int32 [n]); a frame whose status is not OK is zeros."""
    return _streams.decode_host("sfe_jpeg_", streams, R, B, ctx)


def coefficients_host(streams, R, B, ctx=None):
    """Diagnostic: the dequantised coefficient blocks the device IDCT consumes, int32 [n, cap_blocks, 64] (natural
    order, blocks in decode order), and the status array."""
    ctx = ctx or _lib.default_context()
    buf, off = _streams.packed(streams)
    n = len(off) - 1
    info = inspect((buf, off))
    cap = 1
    for st, h, w, nc, samp, _ in info:
        if st == OK:
            hm, vm = {GRAY: (1, 1), S444: (1, 1), S422: (2, 1), S420: (2, 2)}[samp]
            bpm = 1 if nc == 1 else hm * vm + 2
            cap = max(cap, -(-w // (8 * hm)) * -(-h // (8 * vm)) * bpm)
    coef = np.zeros((n, cap, 64), np.int32)
    st = np.zeros(n, np.int32)
    _lib.check(ctx.lib.sfe_jpeg_coefficients_host(ctx.handle, _lib.ptr(buf), _lib.ptr(off), n, int(R), int(B), cap,
                                                  _lib.ptr(coef), _lib.ptr(st)), "sfe_jpeg_coefficients_host")
    return coef, st


STAGES = ("unstuff", "entropy", "idct_color")


def set_timing(enable=True, ctx=None):
    """Per-stage device timing of the decoders on this context (CUDA events around every chunk's kernels)."""
    _streams.set_timing("sfe_jpeg_", enable, ctx)


def get_timing(ctx=None):
    """dict stage -> (total ms, number of timed intervals) since set_timing(True)."""
    return _streams.get_timing("sfe_jpeg_", STAGES, ctx)
