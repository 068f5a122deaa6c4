"""CPU: the argument checks the JPEG and PNG decoders share (csrc/stream_decode.cu) reject a bad call with SFE_ERR_ARG
before any device call, and both codecs word the rejection the same way."""
import ctypes

import numpy as np
import pytest

from sonar_slam_b200 import _lib

SFE_ERR_ARG = -1
CODECS = ("jpeg", "png")
DECREASING = np.array([0, 8, 4], np.int64)
GOOD = np.array([0, 8, 16], np.int64)
# Stands in for an sfe_ctx: the checks must reject the call before they read the context or touch a device.
UNTOUCHED = np.zeros(4096, np.uint8)


def _call(codec, entry, ctx, offsets):
    lib = _lib.load()
    name = f"sfe_{codec}_{entry}"
    buf = np.zeros(16, np.uint8)
    n = len(offsets) - 1
    if entry == "inspect_host":
        rc = getattr(lib, name)(_lib.ptr(buf), _lib.ptr(offsets), n, _lib.ptr(np.zeros((n, 8), np.int32)))
    else:
        out, st = np.zeros((n, 4, 4), np.uint8), np.zeros(n, np.int32)
        rc = getattr(lib, name)(ctx, _lib.ptr(buf), _lib.ptr(offsets), n, 4, 4, _lib.ptr(out), _lib.ptr(st))
    return rc, lib.sfe_last_error().decode().replace(name, "<entry>")


@pytest.mark.parametrize("entry,ctx,offsets,message", [
    ("inspect_host", None, DECREASING, "<entry>: offsets must be non-decreasing"),
    ("decode_host", ctypes.c_void_p(UNTOUCHED.ctypes.data), DECREASING, "<entry>: offsets must be non-decreasing"),
    ("decode_to_dev", ctypes.c_void_p(UNTOUCHED.ctypes.data), DECREASING, "<entry>: offsets must be non-decreasing"),
    ("decode_host", None, GOOD, "<entry>: null argument"),
    ("decode_to_dev", None, GOOD, "<entry>: null argument"),
])
def test_both_codecs_reject_bad_calls_alike_before_any_device_call(entry, ctx, offsets, message):
    got = [_call(codec, entry, ctx, offsets) for codec in CODECS]
    assert got == [(SFE_ERR_ARG, message)] * len(CODECS)
    assert not UNTOUCHED.any()
