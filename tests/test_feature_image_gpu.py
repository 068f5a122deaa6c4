"""GPU: the device feature image (csrc/featx.cu: feature_image_kernel) equals the reference's
cv2.applyColorMap(cv2.remap(img, map_x, map_y, INTER_LINEAR), 2) (feature_extraction.py:226-228) bit for bit, standalone,
from every front-end run flavour and from FeatureExtraction; the front end's numeric results do not depend on it."""
import ctypes
import hashlib
import types

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import feature_image_ref as fir  # noqa: E402
from oracle import featx_ref, jpeg_ref  # noqa: E402
from sonar_slam_b200 import _lib, feature_image, synth  # noqa: E402

pytestmark = pytest.mark.gpu

BEARINGS = {"uniform": synth.bearings_uniform, "oculus": synth.bearings_oculus}
# (rows, cols, R, B): cols odd, rows * cols * 3 not a multiple of 16 (frame bases not 16-B aligned), R and B not
# multiples of 32; one geometry has a tile count above one
ODD_GEOMETRIES = [(64, 77, 45, 37), (33, 31, 17, 50), (129, 127, 100, 96), (5, 3, 1, 1), (40, 41, 2, 3)]
LUTS = {"jet": feature_image.JET, "identity": fir.identity_lut()}
N = 19  # more than one CTA's frame group (8), with a tail


def _maps(ctx, mx, my, R, B):
    return _lib.Maps(ctx, mx, my, R, B, 10.0, 10.0)


def _want(frames, mx, my, lut):
    return np.stack([fir.cv2_feature_image(f, mx, my, None if lut is feature_image.JET else lut) for f in frames])


@pytest.mark.parametrize("lut", sorted(LUTS))
@pytest.mark.parametrize("tag", sorted(BEARINGS))
def test_sonar_geometry_equals_cv2(gpu_ctx, tag, lut):
    import torch
    from sonar_slam_b200 import ops
    geo = featx_ref.Geometry(30.0 / 512, 512, BEARINGS[tag](512))
    maps = _maps(gpu_ctx, geo.map_x, geo.map_y, 512, 512)
    rng = np.random.default_rng(5)
    frames = np.stack([synth.make_frame(s) for s in range(N - 2)] +
                      [rng.integers(0, 256, (512, 512), dtype=np.uint8), np.full((512, 512), 255, np.uint8)])
    want = _want(frames, geo.map_x, geo.map_y, LUTS[lut])
    got = feature_image.render_host(maps, frames, LUTS[lut], ctx=gpu_ctx)
    assert np.array_equal(got, want)
    dev = ops.feature_image(torch.from_numpy(frames).cuda(), maps, LUTS[lut], ctx=gpu_ctx)
    gpu_ctx.sync()
    assert np.array_equal(dev.cpu().numpy(), want)
    one = feature_image.render_host(maps, frames[3], LUTS[lut], ctx=gpu_ctx)
    assert np.array_equal(one[0], want[3])


@pytest.mark.parametrize("geometry", ODD_GEOMETRIES)
def test_edge_maps_and_odd_geometries_equal_cv2(gpu_ctx, geometry):
    rows, cols, R, B = geometry
    rng = np.random.default_rng(rows)
    for seed in range(2):
        mx, my = fir.edge_maps(rows, cols, R, B, seed)
        maps = _maps(gpu_ctx, mx, my, R, B)
        frames = rng.integers(0, 256, (N, R, B), dtype=np.uint8)
        for lut in LUTS.values():
            got = feature_image.render_host(maps, frames, lut, ctx=gpu_ctx)
            assert np.array_equal(got, _want(frames, mx, my, lut)), (geometry, seed)


def test_golden_digests(gpu_ctx, golden_dir):
    g = np.load(f"{golden_dir}/feature_img.npz")
    img = synth.make_frame(1)
    for tag in BEARINGS:
        geo = featx_ref.Geometry(30.0 / 512, 512, BEARINGS[tag](512))
        vis = feature_image.render_host(_maps(gpu_ctx, geo.map_x, geo.map_y, 512, 512), img, ctx=gpu_ctx)[0]
        assert hashlib.sha256(vis.tobytes()).hexdigest() == g[tag + "_sha256"], tag


def _frontend(ctx, n, **kw):
    from sonar_slam_b200 import pipeline
    d = synth.make_trajectory_frames(n, seed=2)
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _maps(ctx, geo.map_x, geo.map_y, 512, 512)
    return d["frames"].numpy(), d["poses_odom"], geo, maps, (lambda: pipeline.FrontEnd(ctx, maps, max_frames=n, **kw))


KEYS = ("T", "iterations", "inliers", "status", "npoints")


@pytest.mark.parametrize("flavour", ["host", "dev", "jpeg", "png"])
@pytest.mark.parametrize("mode", ["cold", "carry"])
def test_frontend_images(gpu_ctx, flavour, mode):
    import torch
    n = 40
    frames, poses, geo, maps, make = _frontend(gpu_ctx, n, min_points=30)
    if flavour == "jpeg":
        inputs = [jpeg_ref.encode(f, 90) for f in frames]
        decoded = np.stack([jpeg_ref.cv2_gray(b) for b in inputs])
    elif flavour == "png":
        inputs = [cv2.imencode(".png", f)[1].tobytes() for f in frames]
        decoded = frames
    else:
        inputs, decoded = frames, frames
    want = feature_image.render_host(maps, decoded, ctx=gpu_ctx)
    for k in (0, 17, n - 1):
        assert np.array_equal(want[k], fir.cv2_feature_image(decoded[k], geo.map_x, geo.map_y))
    pieces = (slice(0, 25), slice(25, n)) if mode == "carry" else (slice(0, n),)

    def run(fe, s, chunk, images):
        if flavour == "dev":
            t = torch.from_numpy(np.ascontiguousarray(frames[s])).cuda()
            gpu_ctx.sync()
            img_t = None if images is None else torch.empty(images.shape, dtype=torch.uint8, device="cuda")
            fe.run_dev(t.data_ptr(), poses[s], len(t), images=img_t)
            r = fe.results_dev()
            m = len(t)
            out = dict(T=gpu_ctx.to_host(r["T"], (m, 3, 3), np.float32),
                       iterations=gpu_ctx.to_host(r["iterations"], m, np.int32),
                       inliers=gpu_ctx.to_host(r["inliers"], m, np.int32),
                       status=gpu_ctx.to_host(r["status"], m, np.int32))
            out["npoints"] = gpu_ctx.to_host(r["cloud_count"], m, np.int32)
            if images is not None:
                images[...] = img_t.cpu().numpy()
            return out
        fn = dict(host=fe.run_host, jpeg=fe.run_jpeg_host, png=fe.run_png_host)[flavour]
        src = inputs[s]
        return fn(src, poses[s], chunk_frames=chunk, images=images)

    for chunk in (7, 16, 256):
        a, b = make(), make()
        if mode == "carry":
            a.set_carry(True), b.set_carry(True)
        for s in pieces:
            images = np.full((s.stop - s.start, maps.rows, maps.cols, 3), 7, np.uint8)
            ra, rb = run(a, s, chunk, None), run(b, s, chunk, images)
            for key in KEYS:
                assert np.array_equal(ra[key], rb[key]), (flavour, mode, chunk, key)
            assert np.array_equal(images, want[s]), (flavour, mode, chunk)
        assert (ra["status"] == 0).sum() > 5
        assert (run(b, pieces[-1], chunk, None)["status"] >= 0).all()  # images are off again after a call


def test_feature_extraction_render_feature_img(gpu_ctx):
    from sonar_slam_b200.bruce_slam.feature_extraction import FeatureExtraction
    for compressed in (False, True):
        fe = FeatureExtraction()
        fe.init_node({"CFAR": {"Ntc": 40, "Ngc": 10, "Pfa": 0.1, "rank": 10, "alg": "SOCA"},
                      "filter": {"threshold": 65, "resolution": 0.5, "radius": 1.0, "min_points": 5, "skip": 2},
                      "compressed_images": compressed})
        fe.decode_on_device = compressed
        bearings = synth.bearings_oculus(512)
        img = synth.make_frame(6)
        data = cv2.imencode(".png", img)[1].tobytes() if compressed else img
        msg = lambda pid: types.SimpleNamespace(ping_id=pid, ping=types.SimpleNamespace(data=data) if compressed else img,
                                                image=None if compressed else img, range_resolution=30.0 / 512,
                                                num_ranges=512, bearings=bearings, header=None)
        pts_off = fe.callback(msg(0))
        assert fe.feature_img is None
        fe.render_feature_img = True
        pts_on = fe.callback(msg(0))
        assert np.array_equal(pts_on, pts_off)
        want = cv2.applyColorMap(cv2.remap(img, fe.map_x, fe.map_y, cv2.INTER_LINEAR), 2)  # :226-227
        assert fe.feature_img.dtype == np.uint8 and np.array_equal(fe.feature_img, want)
        m = fe.feature_img_msg
        assert (m.encoding, m.height, m.width, m.step) == ("bgr8", fe.rows, fe.cols, 3 * fe.cols)
        assert m.data == want.tobytes()
        fe.callback(msg(1))  # skipped ping
        assert fe.feature_img is None


def test_error_messages(gpu_ctx):
    import torch
    from sonar_slam_b200 import ops
    frames, poses, geo, maps, make = _frontend(gpu_ctx, 4)
    with pytest.raises(ValueError, match=r"frames must be \[n, 512, 512\]"):
        feature_image.render_host(maps, np.zeros((2, 256, 512), np.uint8), ctx=gpu_ctx)
    with pytest.raises(ValueError, match=r"frames must be \[n, 512, 512\]"):
        ops.feature_image(torch.zeros((2, 512, 256), dtype=torch.uint8, device="cuda"), maps, ctx=gpu_ctx)
    with pytest.raises(ValueError, match="colour table"):
        feature_image.render_host(maps, frames, np.zeros((255, 3), np.uint8), ctx=gpu_ctx)
    lib = gpu_ctx.lib
    dummy = ctypes.c_void_p(16)
    rc = lib.sfe_feature_image_dev(gpu_ctx.handle, maps.handle, dummy, 1, None, dummy)
    assert rc == -1 and b"null frames, table or output pointer" in lib.sfe_last_error()
    rc = lib.sfe_feature_image_dev(gpu_ctx.handle, maps.handle, dummy, 2 ** 31 - 1, _lib.ptr(feature_image.lut_array(
        feature_image.JET)), dummy)
    assert rc == -1 and b"too many for one call" in lib.sfe_last_error()
    rc = lib.sfe_feature_image_host(gpu_ctx.handle, None, dummy, 1, None, dummy)
    assert rc == -1 and b"null context or maps" in lib.sfe_last_error()
    fe = make()
    n = len(frames)
    with pytest.raises(ValueError, match="images must be"):
        fe.run_host(frames, poses, images=np.zeros((n, 10, 10, 3), np.uint8))
    with pytest.raises(ValueError, match="images must be a contiguous CUDA"):
        fe.run_dev(torch.from_numpy(frames).cuda().data_ptr(), poses, n,
                   images=np.zeros((n, maps.rows, maps.cols, 3), np.uint8))
    host_dst = np.zeros((n, maps.rows, maps.cols, 3), np.uint8)
    _lib.check(lib.sfe_frontend_set_feature_images(fe.handle, _lib.ptr(feature_image.lut_array(feature_image.JET)),
                                                   _lib.ptr(host_dst), 1))
    with pytest.raises(_lib.SonarFEError, match="run_dev: feature images are set to go to host memory"):
        fe.run_dev(torch.from_numpy(frames).cuda().data_ptr(), poses, n)
    rc = lib.sfe_frontend_set_feature_images(fe.handle, None, _lib.ptr(host_dst), 1)
    assert rc == -1 and b"null colour table" in lib.sfe_last_error()
    dev_dst = torch.empty((n, maps.rows, maps.cols, 3), dtype=torch.uint8, device="cuda")
    _lib.check(lib.sfe_frontend_set_feature_images(fe.handle, _lib.ptr(feature_image.lut_array(feature_image.JET)),
                                                   ctypes.c_void_p(dev_dst.data_ptr()), 0))
    with pytest.raises(_lib.SonarFEError, match="run_host: feature images are set to go to device memory"):
        fe.run_host(frames, poses)
    _lib.check(lib.sfe_frontend_set_feature_images(fe.handle, None, None, 0))
    with pytest.raises(_lib.SonarFEError, match="exceed max_frames"):
        fe.run_host(np.concatenate([frames, frames]), np.concatenate([poses, poses]),
                    images=np.zeros((2 * n, maps.rows, maps.cols, 3), np.uint8))
    assert (fe.run_host(frames, poses)["status"] >= 0).all()
