"""GPU: the device PNG decoder (csrc/png.cu) equals cv2.imdecode(IMREAD_COLOR) + BGR2GRAY -- the reference's decode,
feature_extraction.py:210-213 -- bit for bit, and the front end fed with PNG pings equals the front end fed with the
frames cv2 decodes."""
import hashlib
import itertools

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import featx_ref, jpeg_ref, png_ref  # noqa: E402
from sonar_slam_b200 import png, synth  # noqa: E402

pytestmark = pytest.mark.gpu


def _check(streams, R, B, ctx):
    out, st = png.decode_host(streams, R, B, ctx=ctx)
    for i, b in enumerate(streams):
        assert st[i] == png.OK, (i, png.status_message(st[i]))
        want = png_ref.cv2_gray(b)
        assert np.array_equal(out[i], want), (i, R, B, int((out[i] != want).sum()))
    return out


@pytest.mark.parametrize("size", [(1, 1), (1, 9), (9, 1), (7, 9), (17, 33), (64, 48)])
def test_bit_identity_option_grid(gpu_ctx, size):
    h, w = size
    streams = []
    for k, (rgb, strategy, level, wbits, idat) in enumerate(itertools.product(
            (False, True), list(png_ref.STRATEGIES), (0, 1, 6, 9), (9, 15), (None, 1, -7))):
        img = jpeg_ref.contents(h, w, seed=k)[("synth", "noise", "checker")[k % 3]]
        filters = [(y + k) % 5 for y in range(h)] if k % 2 else k % 5
        streams.append(png_ref.write(png_ref.rgb_of(img) if rgb else img, filters, level, strategy, wbits, idat))
    _check(streams, h, w, gpu_ctx)


def test_bit_identity_every_filter_full_size(gpu_ctx):
    img = synth.make_frame(4)
    rng = np.random.default_rng(2)
    streams = [png_ref.write(img, f) for f in range(5)] + [png_ref.write(img, rng.integers(0, 5, 512))]
    streams += [png_ref.write(png_ref.rgb_of(img), f) for f in (1, 4)]
    streams += [cv2.imencode(".png", synth.make_frame(s))[1].tobytes() for s in range(4)]
    _check(streams, 512, 512, gpu_ctx)


def test_golden_digests(gpu_ctx, golden_dir):
    g = np.load(f"{golden_dir}/png_streams.npz")
    off = g["offsets"]
    for shape in {tuple(s) for s in g["shapes"]}:
        idx = [i for i, s in enumerate(g["shapes"]) if tuple(s) == shape]
        streams = [g["bytes"][off[i]:off[i + 1]].tobytes() for i in idx]
        out, st = png.decode_host(streams, *shape, ctx=gpu_ctx)
        for k, i in enumerate(idx):
            assert st[k] == png.OK and hashlib.sha256(out[k].tobytes()).hexdigest() == g["sha256"][i], g["names"][i]


def test_edge_streams_and_accepted_header_variants(gpu_ctx):
    for name, (h, w, b) in png_ref.edge_streams().items():
        _check([b], h, w, gpu_ctx)
    img = jpeg_ref.contents(64, 48)["synth"]
    ok = [b for b, st in png_ref.rejected_variants(img).values() if st == "OK"]
    _check(ok + [png_ref.over_long(img)], 64, 48, gpu_ctx)


def test_mixed_call_statuses_and_isolation(gpu_ctx):
    """Valid, corrupt (every kind), rejected and over-long streams in one call: each frame gets its status, corrupt
    and rejected frames are zeros and every valid frame is exact."""
    img = jpeg_ref.contents(64, 48, seed=3)["synth"]
    good = [png_ref.write(jpeg_ref.contents(64, 48, seed=s)["synth"], s % 5) for s in range(4)]
    corrupt = list(png_ref.corrupt_variants(img).values())
    rejected = [(b, getattr(png, st)) for b, st in png_ref.rejected_variants(img).values() if st != "OK"]
    batch, want = [], []
    for k, b in enumerate(corrupt):
        batch += [good[k % 4], b]
        want += [png.OK, png.CORRUPT]
    for b, st in rejected:
        batch += [b, png_ref.over_long(img)]
        want += [st, png.OK]
    batch.append(png_ref.write(jpeg_ref.contents(32, 48)["synth"]))
    want.append(png.SIZE)
    out, st = png.decode_host(batch, 64, 48, ctx=gpu_ctx)
    assert st.tolist() == want
    for i, b in enumerate(batch):
        if want[i] == png.OK:
            assert np.array_equal(out[i], png_ref.cv2_gray(b)), i
        else:
            assert not out[i].any(), i


def test_ops_decode_png_device_tensor(gpu_ctx):
    import torch
    from sonar_slam_b200 import ops
    streams = [cv2.imencode(".png", f)[1].tobytes() for f in synth.make_frames(range(3))]
    out, st = ops.decode_png(streams, 512, 512, device=0)
    torch.cuda.synchronize()
    assert out.is_cuda and out.dtype == torch.uint8 and (st == 0).all()
    for i, b in enumerate(streams):
        assert np.array_equal(out[i].cpu().numpy(), png_ref.cv2_gray(b))


def test_large_call_on_cv2_pings(gpu_ctx):
    frames = synth.make_frames(range(16))
    enc = [cv2.imencode(".png", f)[1].tobytes() for f in frames]
    streams = [enc[i % 16] for i in range(4096)]
    out, st = png.decode_host(streams, 512, 512, ctx=gpu_ctx)
    assert (st == png.OK).all()
    rng = np.random.default_rng(7)
    for i in sorted(set(rng.integers(0, 4096, 24).tolist()) | {0, 4095}):
        assert np.array_equal(out[i], frames[i % 16]), i


def _frontend(ctx, n, **kw):
    from sonar_slam_b200 import _lib, pipeline
    d = synth.make_trajectory_frames(n, seed=2)
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    return d["frames"].numpy(), d["poses_odom"], maps, (lambda: pipeline.FrontEnd(ctx, maps, max_frames=n, **kw))


@pytest.mark.parametrize("mode", ["cold", "carry", "plane"])
def test_run_png_host_equals_run_host_on_cv2_frames(gpu_ctx, mode):
    from sonar_slam_b200 import _lib
    kw = dict(min_points=30)
    if mode == "plane":
        kw["icp"] = _lib.IcpParams(minimizer=1, normals_knn=5)
    frames, poses, maps, make = _frontend(gpu_ctx, 40, **kw)
    streams = [cv2.imencode(".png", f)[1].tobytes() if i % 3 else png_ref.write(png_ref.rgb_of(f), i % 5)
               for i, f in enumerate(frames)]
    decoded = np.stack([png_ref.cv2_gray(b) for b in streams])
    keys = ("T", "iterations", "inliers", "status", "npoints")
    for chunk in (7, 16, 256):
        a, b = make(), make()
        if mode == "carry":
            a.set_carry(True), b.set_carry(True)
            ra = [a.run_host(decoded[s], poses[s], chunk_frames=chunk) for s in (slice(0, 25), slice(25, 40))]
            rb = [b.run_png_host(streams[s], poses[s], chunk_frames=chunk) for s in (slice(0, 25), slice(25, 40))]
        else:
            ra, rb = [a.run_host(decoded, poses, chunk_frames=chunk)], [b.run_png_host(streams, poses, chunk)]
        for x, y in zip(ra, rb):
            for k in keys:
                assert np.array_equal(x[k], y[k]), (mode, chunk, k)
        assert (ra[0]["status"] == 0).sum() > 10


def test_run_png_host_names_the_first_bad_frame(gpu_ctx):
    from sonar_slam_b200 import _lib
    frames, poses, maps, make = _frontend(gpu_ctx, 6)
    streams = [cv2.imencode(".png", f)[1].tobytes() for f in frames]
    fe = make()
    with pytest.raises(_lib.SonarFEError, match="frame 3: interlaced"):
        adam7 = png_ref.assemble(512, 512, png_ref.deflate(png_ref.filter_rows(frames[3], 1, 1)), interlace=1)
        fe.run_png_host(streams[:3] + [adam7] + streams[4:], poses)
    with pytest.raises(_lib.SonarFEError, match="frame 4: corrupt"):
        bad = png_ref.corrupt_variants(frames[4])["adler"]
        fe.run_png_host(streams[:4] + [bad] + streams[5:], poses, chunk_frames=2)
    with pytest.raises(_lib.SonarFEError, match="frame 0: not a PNG"):
        fe.run_png_host([jpeg_ref.encode(frames[0], 80)] + streams[1:], poses)
    assert (fe.run_png_host(streams, poses)["status"] >= 0).all()


def test_feature_extraction_decode_on_device(gpu_ctx):
    import types
    from sonar_slam_b200.bruce_slam.feature_extraction import FeatureExtraction
    fe = FeatureExtraction()
    fe.init_node({"CFAR": {"Ntc": 40, "Ngc": 10, "Pfa": 0.1, "rank": 10, "alg": "SOCA"},
                  "filter": {"threshold": 65, "resolution": 0.5, "radius": 1.0, "min_points": 5, "skip": 1},
                  "compressed_images": True})
    img = synth.make_frame(3)
    for b in (cv2.imencode(".png", img)[1].tobytes(), cv2.imencode(".png", png_ref.rgb_of(img))[1].tobytes(),
              png_ref.write(img, png_ref.PAETH), png_ref.corrupt_variants(img)["idat_crc"]):
        msg = types.SimpleNamespace(ping=types.SimpleNamespace(data=b))

        def image(on_device):
            fe.decode_on_device = on_device
            try:
                return fe.ping_image(msg)
            except ValueError as e:                                # cv2.imdecode gave nothing: both paths say so
                return str(e)
        host, dev = image(False), image(True)
        assert type(dev) is type(host)
        assert dev == host if isinstance(host, str) else (dev.dtype == np.uint8 and np.array_equal(dev, host))


def test_stage_timing(gpu_ctx):
    streams = [cv2.imencode(".png", f)[1].tobytes() for f in synth.make_frames(range(4))]
    png.set_timing(True, ctx=gpu_ctx)
    png.decode_host(streams, 512, 512, ctx=gpu_ctx)
    t = png.get_timing(ctx=gpu_ctx)
    png.set_timing(False, ctx=gpu_ctx)
    assert list(t) == list(png.STAGES) and all(ms > 0 and calls == 1 for ms, calls in t.values())
