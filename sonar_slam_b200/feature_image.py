"""The sonar feature image (feature_extraction.py:226-228) on the device.

The reference publishes, for every processed ping,

    vis_img = cv2.applyColorMap(cv2.remap(img, map_x, map_y, cv2.INTER_LINEAR), 2)     # COLORMAP_JET, bgr8

`render_host` computes the same image bit for bit on the GPU (include/sonarfe.h: sfe_feature_image_host) for a batch
of polar frames; `ops.feature_image` is the device-tensor form and the front end can write the images of the frames it
processes (`FrontEnd.run_*(..., images=...)`).  cv2 is not needed at run time: `JET` is OpenCV's COLORMAP_JET table.
"""
import numpy as np

from . import _lib


def _jet():
    """OpenCV's COLORMAP_JET as the 256-entry bgr8 table cv2.applyColorMap uses: each channel ramps by 4 per entry
    between plateaus of 0 and 255 (OpenCV's breakpoint values times 255, rounded); the blue ramp down ends at 1."""
    up = lambda a: np.arange(a, a + 4 * 63 + 1, 4)          # 64 entries a, a+4, ..., a+252
    down = lambda a: np.arange(a, a - 4 * 63 - 1, -4)
    f = np.full(64, 255)
    b = np.r_[np.arange(128, 253, 4), np.full(64, 255), down(254)[:63], 1, np.zeros(96, int)]
    g = np.r_[np.zeros(33, int), up(4)[:63], f, down(252)[:63], np.zeros(33, int)]
    r = np.r_[np.zeros(96, int), up(2), f, down(252)[:32]]
    return np.ascontiguousarray(np.stack([b, g, r], 1).astype(np.uint8))


JET = _jet()
JET.setflags(write=False)


def lut_array(lut):
    """A colour table as the library takes it: C-contiguous uint8 [256, 3] (B, G, R per grey level)."""
    lut = np.ascontiguousarray(lut, np.uint8)
    if lut.shape != (256, 3):
        raise ValueError(f"feature image: the colour table must be uint8 [256, 3], got {lut.shape}")
    return lut


def render_host(maps, frames, lut=JET, ctx=None, out=None):
    """Feature images of polar frames in host memory.  maps: _lib.Maps of the geometry; frames: uint8 [n, R, B] (or
    [R, B]).  Returns uint8 [n, rows, cols, 3] bgr8 (in `out` when given)."""
    frames = np.ascontiguousarray(frames, np.uint8)
    if frames.ndim == 2:
        frames = frames[None]
    if frames.ndim != 3 or frames.shape[1:] != (maps.R, maps.B):
        raise ValueError(f"feature image: frames must be [n, {maps.R}, {maps.B}] for these maps, got {frames.shape}")
    lut = lut_array(lut)
    n = len(frames)
    if out is None:
        out = np.empty((n, maps.rows, maps.cols, 3), np.uint8)
    elif out.shape != (n, maps.rows, maps.cols, 3) or out.dtype != np.uint8 or not out.flags["C_CONTIGUOUS"]:
        raise ValueError(f"feature image: out must be C-contiguous uint8 [{n}, {maps.rows}, {maps.cols}, 3]")
    ctx = ctx or _lib.default_context()
    _lib.check(ctx.lib.sfe_feature_image_host(ctx.handle, maps.handle, _lib.ptr(frames), n, _lib.ptr(lut),
                                              _lib.ptr(out)), "sfe_feature_image_host")
    return out
