"""CPU-only: the argument checks of the front end's per-frame geometry (FrontEnd.add_geometry, geometry=) that run
before the library is asked to do anything, and the C entry points' own null checks."""
import ctypes
import types

import numpy as np
import pytest

from sonar_slam_b200 import _lib, pipeline

SFE_ERR_ARG = -1


def _front_end():
    """A FrontEnd with geometries 512 x 512 (id 0) and 384 x 256 (id 1), without a device behind it."""
    fe = object.__new__(pipeline.FrontEnd)
    fe.maps = types.SimpleNamespace(R=512, B=512, rows=512, cols=930)
    fe.geometries = [fe.maps, types.SimpleNamespace(R=384, B=256, rows=384, cols=700)]
    return fe


def test_pack_frames_of_two_geometries():
    fe = _front_end()
    rng = np.random.default_rng(0)
    frames = [rng.integers(0, 256, s, dtype=np.uint8) for s in [(512, 512), (384, 256), (384, 256), (512, 512)]]
    buf, off = fe.pack_frames(frames, np.array([0, 1, 1, 0], np.int32))
    assert off.dtype == np.int64 and list(np.diff(off)) == [512 * 512, 384 * 256, 384 * 256, 512 * 512]
    for i, f in enumerate(frames):
        assert np.array_equal(buf[off[i]:off[i + 1]].reshape(f.shape), f)
    # the packed form is passed through as it is once its offsets are inside the buffer
    b2, o2 = fe.pack_frames((buf, off), None)
    assert b2.ctypes.data == buf.ctypes.data and np.array_equal(o2, off)


def test_frame_shape_must_be_its_geometry():
    fe = _front_end()
    frames = [np.zeros((512, 512), np.uint8), np.zeros((256, 384), np.uint8)]
    with pytest.raises(ValueError, match=r"frame 1 has shape \(256, 384\); its geometry 1 is 384 x 256"):
        fe.pack_frames(frames, np.array([0, 1], np.int32))
    # ids the front end does not have are left to the library, which names them
    buf, off = fe.pack_frames(frames, np.array([0, 5], np.int32))
    assert off[-1] == 512 * 512 + 256 * 384


@pytest.mark.parametrize("off", [[0, 100, 201], [-1, 100, 200], [[0, 100, 200]]])
def test_packed_offsets_must_stay_inside_the_buffer(off):
    fe = _front_end()
    with pytest.raises(ValueError, match="overrun the packed buffer"):
        fe.pack_frames((np.zeros(200, np.uint8), np.array(off, np.int64)), None)


def test_one_geometry_id_per_frame():
    fe = _front_end()
    assert fe._geometry(None, 3) is None
    assert fe._geometry([0, 1, 1], 3).dtype == np.int32
    with pytest.raises(ValueError, match="geometry has 2 ids for 3 frames"):
        fe._geometry([0, 1], 3)


def test_images_take_the_size_of_the_calls_geometry():
    fe = _front_end()
    assert fe._image_maps(None) is fe.maps
    assert fe._image_maps(np.array([1, 1], np.int32)) is fe.geometries[1]
    assert fe._image_maps(np.array([7], np.int32)) is fe.maps      # an unknown id: the library refuses the call


def test_entry_points_refuse_null_arguments():
    lib = _lib.load()
    gid = ctypes.c_int(-5)
    assert lib.sfe_frontend_add_geometry(None, None, ctypes.byref(gid)) == SFE_ERR_ARG
    assert b"null argument" in lib.sfe_last_error() and gid.value == -5
    out = [None] * 5
    assert lib.sfe_frontend_run_dev_geometry(None, None, None, None, 0) == SFE_ERR_ARG
    assert b"null geometry" in lib.sfe_last_error()
    assert lib.sfe_frontend_run_host_geometry(None, None, None, None, None, 0, 0, *out) == SFE_ERR_ARG
    assert b"null offsets / geometry" in lib.sfe_last_error()
    for name in ("sfe_frontend_run_jpeg_host_geometry", "sfe_frontend_run_png_host_geometry"):
        assert getattr(lib, name)(None, None, None, None, None, 0, 0, *out) == SFE_ERR_ARG
        assert b"null geometry" in lib.sfe_last_error()

