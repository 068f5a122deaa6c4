"""PNG-compressed sonar pings decoded on the device (include/sonarfe.h: sfe_png_*; csrc/png.cu).

The reference decodes every ping of a compressed bag with cv2.imdecode(IMREAD_COLOR) + cvtColor(BGR2GRAY)
(feature_extraction.py:210-213).  For 8-bit gray or truecolour, non-interlaced PNG (any deflate content, any row
filter) the device decoder gives the same uint8 frames bit for bit; other streams (palette, alpha, 16-bit, Adam7,
APNG, JPEG ...) get a status naming the reason and stay on the host path.  The chunk list is walked on the host, so
`inspect` needs no GPU.  Streams are packed with jpeg.pack.
"""
from . import _lib, _streams

(OK, NOT_PNG, TRUNCATED, BAD_HEADER, DEPTH, COLORTYPE, INTERLACED, ORIENTATION, ANIMATED, SIZE,
 CORRUPT) = range(11)                                     # SFE_PNG_* status
INFO_FIELDS = ("status", "height", "width", "colour_type", "idat_chunks")
SIGNATURE = b"\x89PNG\r\n\x1a\n"


def status_message(status):
    return _lib.load().sfe_png_status_message(int(status)).decode()


def inspect(streams):
    """Chunk list only (no GPU): int32 [n, 5] rows (status, height, width, colour type, IDAT chunks)."""
    return _streams.inspect("sfe_png_", streams, INFO_FIELDS)


def decode_host(streams, R, B, ctx=None):
    """Decode into host memory: (uint8 [n, R, B], status int32 [n]); a frame whose status is not OK is zeros."""
    return _streams.decode_host("sfe_png_", streams, R, B, ctx)


STAGES = ("check", "inflate", "unfilter")


def set_timing(enable=True, ctx=None):
    """Per-stage device timing of the decoder on this context (CUDA events around every chunk's kernels)."""
    _streams.set_timing("sfe_png_", enable, ctx)


def get_timing(ctx=None):
    """dict stage -> (total ms, number of timed intervals) since set_timing(True)."""
    return _streams.get_timing("sfe_png_", STAGES, ctx)
