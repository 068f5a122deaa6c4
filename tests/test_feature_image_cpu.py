"""CPU: the feature image's colour table and integer remap model (oracle/feature_image_ref.py) against the real cv2, the
sensor_msgs/Image mirror, and the digests captured from the reference's own callback (tests/golden/feature_img.npz)."""
import hashlib

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import feature_image_ref as fir  # noqa: E402
from oracle import featx_ref  # noqa: E402
from sonar_slam_b200 import feature_image, synth  # noqa: E402
from sonar_slam_b200.bruce_slam import conversions  # noqa: E402

BEARINGS = {"uniform": synth.bearings_uniform, "oculus": synth.bearings_oculus}
# (rows, cols, R, B): cols odd, rows * cols not a multiple of 16, R and B not multiples of 32
ODD_GEOMETRIES = [(64, 77, 45, 37), (33, 31, 17, 50), (129, 127, 100, 96), (5, 3, 1, 1), (40, 41, 2, 3)]


def test_jet_is_cv2_colormap_jet():
    want = cv2.applyColorMap(np.arange(256, dtype=np.uint8)[None], 2)[0]
    assert feature_image.JET.dtype == np.uint8 and np.array_equal(feature_image.JET, want)


@pytest.mark.parametrize("tag", sorted(BEARINGS))
def test_model_equals_cv2_on_sonar_geometry(tag):
    geo = featx_ref.Geometry(30.0 / 512, 512, BEARINGS[tag](512))
    rng = np.random.default_rng(3)
    frames = [synth.make_frame(1), rng.integers(0, 256, (512, 512), dtype=np.uint8),
              np.clip(rng.gamma(2.0, 40.0, (512, 512)), 0, 255).astype(np.uint8)]
    for img in frames:
        want = cv2.remap(img, geo.map_x, geo.map_y, cv2.INTER_LINEAR)
        assert np.array_equal(fir.remap_image_model(img, geo.map_x, geo.map_y), want)
    img = frames[0]
    assert np.array_equal(fir.feature_image_model(img, geo.map_x, geo.map_y, feature_image.JET),
                          fir.cv2_feature_image(img, geo.map_x, geo.map_y))


@pytest.mark.parametrize("geometry", ODD_GEOMETRIES)
def test_model_equals_cv2_on_edge_maps(geometry):
    rows, cols, R, B = geometry
    rng = np.random.default_rng(rows)
    for seed in range(3):
        mx, my = fir.edge_maps(rows, cols, R, B, seed)
        if rows * cols > 1000:
            assert np.isnan(mx).any() and np.isinf(my).any() and (np.abs(mx) > 32768).any()
        img = rng.integers(0, 256, (R, B), dtype=np.uint8)
        assert np.array_equal(fir.remap_image_model(img, mx, my), cv2.remap(img, mx, my, cv2.INTER_LINEAR))
        assert np.array_equal(fir.feature_image_model(img, mx, my, feature_image.JET),
                              fir.cv2_feature_image(img, mx, my))


def test_non_convertible_coordinates_give_zero():
    img = np.full((8, 8), 200, np.uint8)
    vals = np.array([np.nan, np.inf, -np.inf, 1e10, -1e10, 3e9, 70000.0, -70000.0], np.float32)
    mx = np.r_[vals, np.full(len(vals), 3.0, np.float32)][None]
    my = np.r_[np.full(len(vals), 3.0, np.float32), vals][None]
    assert not cv2.remap(img, mx, my, cv2.INTER_LINEAR).any()
    assert not fir.remap_image_model(img, mx, my).any()


def test_numpy_to_image_mirror():
    arr = np.arange(2 * 5 * 3, dtype=np.uint8).reshape(2, 5, 3)
    msg = conversions.numpy_to_image(arr, "bgr8")
    assert msg._type == "sensor_msgs/Image" and msg.encoding == "bgr8"
    assert (msg.height, msg.width, msg.step, msg.is_bigendian) == (2, 5, 15, False)
    assert msg.data == arr.tobytes()
    assert np.array_equal(np.frombuffer(msg.data, np.uint8).reshape(msg.height, msg.step // 3, 3), arr)
    mono = conversions.numpy_to_image(np.asfortranarray(np.arange(12, dtype=np.uint16).reshape(3, 4)), "mono16")
    assert (mono.height, mono.width, mono.step) == (3, 4, 8) and mono.data == np.arange(12, dtype=np.uint16).tobytes()
    for bad in ((arr, "mono8"), (arr.astype(np.float32), "bgr8"), (arr, "xyz"), (arr[None], "bgr8")):
        with pytest.raises(TypeError):
            conversions.numpy_to_image(*bad)


def test_model_reproduces_reference_callback_digests(golden_dir):
    g = np.load(f"{golden_dir}/feature_img.npz")
    img = synth.make_frame(1)
    for tag in BEARINGS:
        geo = featx_ref.Geometry(30.0 / 512, 512, BEARINGS[tag](512))
        assert hashlib.sha256(geo.map_x.tobytes()).hexdigest() == g[tag + "_map_x_sha256"]
        assert hashlib.sha256(geo.map_y.tobytes()).hexdigest() == g[tag + "_map_y_sha256"]
        vis = fir.feature_image_model(img, geo.map_x, geo.map_y, feature_image.JET)
        assert vis.shape == tuple(g[tag + "_shape"])
        assert np.array_equal(vis[::17, ::23], g[tag + "_sample"])
        assert hashlib.sha256(vis.tobytes()).hexdigest() == g[tag + "_sha256"]
