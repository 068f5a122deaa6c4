"""TEST INFRASTRUCTURE ONLY -- CPU oracle for the sonar feature image (feature_extraction.py:226-228):

    vis_img = cv2.applyColorMap(cv2.remap(img, map_x, map_y, cv2.INTER_LINEAR), 2)

`remap_image_model` is featx_ref.remap_mask_model's integer rule for any uint8 image plus what cv2 does with map
coordinates it cannot convert (NaN, +-inf, |map * 32| >= 1e9: the pixel is 0); `feature_image_model` adds the colour
table look-up.  The CUDA kernel (csrc/featx.cu: feature_image_kernel) implements the same rule; the tests check
model == cv2 == GPU, with the real cv2 as the oracle.  `edge_maps` builds sampling maps that exercise every branch.
"""
import numpy as np


def remap_image_model(img, map_x, map_y):
    """Integer model of cv2.remap(img, map_x, map_y, INTER_LINEAR) for a uint8 [R, B] image (constant-0 border):
    coordinates quantised to 1/32 px with round-half-even, the integer part saturated to int16, weights
    (32-fx)(32-fy), fx(32-fy), (32-fx)fy, fx*fy, result (32 * sum + 2^14) >> 15; a coordinate that is NaN, infinite
    or at least 1e9 in magnitude once multiplied by 32 gives 0."""
    img = np.asarray(img, np.uint8)
    R, B = img.shape
    mx = np.asarray(map_x, np.float32) * np.float32(32)
    my = np.asarray(map_y, np.float32) * np.float32(32)
    with np.errstate(invalid="ignore"):
        dead = ~((np.abs(mx) < 1e9) & (np.abs(my) < 1e9))
    sx = np.rint(np.where(dead, 0, mx)).astype(np.int64)
    sy = np.rint(np.where(dead, 0, my)).astype(np.int64)
    ix, iy = np.clip(sx >> 5, -32768, 32767), np.clip(sy >> 5, -32768, 32767)
    fx, fy = sx & 31, sy & 31
    acc = np.zeros(mx.shape, np.int64)
    for dy, dx, w in ((0, 0, (32 - fx) * (32 - fy)), (0, 1, fx * (32 - fy)), (1, 0, (32 - fx) * fy), (1, 1, fx * fy)):
        yy, xx = iy + dy, ix + dx
        ok = (yy >= 0) & (yy < R) & (xx >= 0) & (xx < B)
        v = np.zeros(mx.shape, np.int64)
        v[ok] = img[yy[ok], xx[ok]]
        acc += w * v
    out = ((32 * acc + 16384) >> 15).astype(np.uint8)
    out[dead] = 0
    return out


def feature_image_model(img, map_x, map_y, lut):
    """bgr8 [rows, cols, 3] = lut[remap_image_model(img, map_x, map_y)]."""
    return np.asarray(lut, np.uint8)[remap_image_model(img, map_x, map_y)]


def cv2_feature_image(img, map_x, map_y, lut=None):
    """The reference's lines :226-227 through the real cv2; with `lut`, cv2.LUT of the remapped grey image instead of
    COLORMAP_JET (the same look-up, any table)."""
    import cv2
    g = cv2.remap(np.ascontiguousarray(img, np.uint8), np.asarray(map_x, np.float32), np.asarray(map_y, np.float32),
                  cv2.INTER_LINEAR)
    if lut is None:
        return cv2.applyColorMap(g, 2)
    lut = np.asarray(lut, np.uint8)
    return np.ascontiguousarray(lut[g])


def edge_maps(rows, cols, R, B, seed=0):
    """Hand-built float32 maps for an R x B polar image: coordinates inside, negative and past the edges, cvRound ties
    at k/64, int16 saturation, NaN, +-inf and values too large to convert, mixed per pixel."""
    rng = np.random.default_rng(seed)
    n = rows * cols
    mx = rng.uniform(-3.0, B + 2.0, n)
    my = rng.uniform(-3.0, R + 2.0, n)
    kind = rng.integers(0, 8, n)
    ties = lambda hi, m: np.floor(rng.uniform(-2, hi + 1, m)) + rng.integers(0, 32, m) / 32.0 + 1 / 64.0
    k = kind == 1  # exact ties at k/64 (x * 32 ends in .5 -> round half to even)
    mx[k], my[k] = ties(B, k.sum()), ties(R, k.sum())
    k = kind == 2  # just inside / outside the last row and column, and around -1
    mx[k] = rng.choice([-1.0, -0.999, -0.5, -1 / 64.0, 0.0, B - 1.0, B - 1 + 1 / 64.0, B - 0.5, B - 1 / 64.0, B * 1.0],
                       k.sum())
    my[k] = rng.choice([-1.0, -0.5, -1 / 64.0, 0.0, R - 1.0, R - 1 + 1 / 64.0, R - 0.5, R * 1.0], k.sum())
    special = np.array([np.nan, np.inf, -np.inf, 1e10, -1e10, 3e9, -3e9, 1e9 / 32, -1e9 / 32, 1.5e9 / 32, 70000.0,
                        -70000.0, 32767.0, 32767.9, -32768.0, -32769.5, 40000.0, 1100.0, -1100.0])
    k = kind == 3  # int16 saturation, non-finite and huge values in x, y or both
    mx[k] = rng.choice(special, k.sum())
    k = kind == 4
    my[k] = rng.choice(special, k.sum())
    k = kind == 5
    mx[k], my[k] = rng.choice(special, k.sum()), rng.choice(special, k.sum())
    return mx.astype(np.float32).reshape(rows, cols), my.astype(np.float32).reshape(rows, cols)


def identity_lut():
    """uint8 [256, 3] with every channel equal to the grey level: the image is the remap itself."""
    return np.repeat(np.arange(256, dtype=np.uint8)[:, None], 3, 1)
