"""GPU: the device JPEG decoder (csrc/jpeg.cu) equals cv2.imdecode(IMREAD_COLOR) + BGR2GRAY -- the reference's decode,
feature_extraction.py:210-213 -- bit for bit, and the front end fed with compressed pings equals the front end fed
with the frames cv2 decodes."""
import hashlib
import itertools

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import featx_ref, jpeg_ref  # noqa: E402
from sonar_slam_b200 import jpeg, synth  # noqa: E402

pytestmark = pytest.mark.gpu

QUALITIES = (1, 5, 10, 25, 50, 75, 80, 90, 95, 100)
RESTARTS = (0, 1, 3, 17)


def _check(streams, R, B, ctx):
    out, st = jpeg.decode_host(streams, R, B, ctx=ctx)
    for i, b in enumerate(streams):
        assert st[i] == jpeg.OK, (i, jpeg.status_message(st[i]))
        want = jpeg_ref.cv2_gray(b)
        assert np.array_equal(out[i], want), (i, R, B, int((out[i] != want).sum()))
    return out


@pytest.mark.parametrize("size", [(1, 1), (7, 9), (8, 8), (16, 16), (17, 33)])
def test_bit_identity_small_sizes_full_grid(gpu_ctx, size):
    h, w = size
    streams = [jpeg_ref.encode(img, q, samp, opt, ri)
               for img in jpeg_ref.contents(h, w, seed=h * 7 + w).values()
               for q, samp, opt, ri in itertools.product(QUALITIES, jpeg_ref.SAMPLINGS, (False, True), RESTARTS)]
    assert len(streams) == 5 * 10 * 4 * 2 * 4
    _check(streams, h, w, gpu_ctx)


@pytest.mark.parametrize("size", [(511, 509), (512, 512)])
def test_bit_identity_full_size_frames(gpu_ctx, size):
    h, w = size
    streams = []
    for k, (q, samp) in enumerate(itertools.product(QUALITIES, jpeg_ref.SAMPLINGS)):
        for name, img in jpeg_ref.contents(h, w, seed=k).items():
            streams.append(jpeg_ref.encode(img, q, samp, (k + len(name)) % 2 == 1, RESTARTS[(k + len(name)) % 4]))
    _check(streams, h, w, gpu_ctx)


def test_golden_digests(gpu_ctx, golden_dir):
    g = np.load(f"{golden_dir}/jpeg_streams.npz")
    off = g["offsets"]
    for shape in {tuple(s) for s in g["shapes"]}:
        idx = [i for i, s in enumerate(g["shapes"]) if tuple(s) == shape]
        streams = [g["bytes"][off[i]:off[i + 1]].tobytes() for i in idx]
        out, st = jpeg.decode_host(streams, *shape, ctx=gpu_ctx)
        for k, i in enumerate(idx):
            assert st[k] == jpeg.OK and hashlib.sha256(out[k].tobytes()).hexdigest() == g["sha256"][i], g["names"][i]


def test_coefficients_equal_the_oracle(gpu_ctx):
    streams = [jpeg_ref.encode(img, q, samp, opt, ri)
               for img in jpeg_ref.contents(17, 33, seed=4).values()
               for q, samp, opt, ri in [(5, "gray", 0, 0), (50, "444", 1, 1), (90, "422", 0, 3), (100, "420", 1, 17)]]
    coef, st = jpeg.coefficients_host(streams, 17, 33, ctx=gpu_ctx)
    for i, b in enumerate(streams):
        want = jpeg_ref.coefficients(b)[0]
        assert st[i] == jpeg.OK
        assert np.array_equal(coef[i, :len(want)], want) and not coef[i, len(want):].any(), i


def test_mixed_batch_equals_single_calls_and_batch_of_one(gpu_ctx):
    rng = np.random.default_rng(5)
    frames = synth.make_frames(range(8))
    streams = [jpeg_ref.encode(frames[i % 8], int(rng.integers(1, 101)), jpeg_ref.SAMPLINGS[i % 4], i % 3 == 0,
                               RESTARTS[i % 4]) for i in range(4096)]
    out, st = jpeg.decode_host(streams, 512, 512, ctx=gpu_ctx)
    assert (st == jpeg.OK).all()
    for i in list(range(12)) + [1000, 2047, 4095]:
        one, s1 = jpeg.decode_host([streams[i]], 512, 512, ctx=gpu_ctx)
        assert s1[0] == jpeg.OK and np.array_equal(one[0], out[i]), i
        assert np.array_equal(out[i], jpeg_ref.cv2_gray(streams[i])), i


def test_corrupt_streams_fail_alone(gpu_ctx):
    frames = synth.make_frames(range(6))
    streams = [jpeg_ref.encode(frames[i], 80, jpeg_ref.SAMPLINGS[i % 4], False, RESTARTS[i % 4]) for i in range(6)]
    bad = list(streams)
    ecs = jpeg_ref.parse(streams[1])["ecs"]
    bad[1] = streams[1][:ecs + (len(streams[1]) - ecs) // 2]                     # truncated: out of data
    ecs = jpeg_ref.parse(streams[2])["ecs"]
    mid = ecs + (len(streams[2]) - ecs) // 3
    bad[2] = streams[2][:mid] + b"\xff\x00" * 8 + streams[2][mid + 16:]           # 64 one bits: no valid code
    ecs = jpeg_ref.parse(streams[3])["ecs"]
    bad[3] = streams[3][:ecs + 40]                                               # restart segments missing
    out, st = jpeg.decode_host(bad, 512, 512, ctx=gpu_ctx)
    assert st.tolist() == [jpeg.OK, jpeg.CORRUPT, jpeg.CORRUPT, jpeg.CORRUPT, jpeg.OK, jpeg.OK]
    for i in (0, 4, 5):
        assert np.array_equal(out[i], jpeg_ref.cv2_gray(streams[i])), i
    assert not out[1:4].any()
    # rejected streams and a wrong frame size get their status too
    out, st = jpeg.decode_host([streams[0], cv2.imencode(".png", frames[0])[1].tobytes(), streams[4]], 512, 256,
                               ctx=gpu_ctx)
    assert st.tolist() == [jpeg.SIZE, jpeg.NOT_JPEG, jpeg.SIZE] and not out.any()


def test_ops_decode_jpeg_device_tensor(gpu_ctx):
    import torch
    from sonar_slam_b200 import ops
    frames = synth.make_frames(range(3))
    streams = [jpeg_ref.encode(f, 80) for f in frames]
    out, st = ops.decode_jpeg(streams, 512, 512, device=0)
    torch.cuda.synchronize()
    assert out.is_cuda and out.dtype == torch.uint8 and (st == 0).all()
    for i, b in enumerate(streams):
        assert np.array_equal(out[i].cpu().numpy(), jpeg_ref.cv2_gray(b))


def _frontend(ctx, n, **kw):
    from sonar_slam_b200 import _lib, pipeline
    d = synth.make_trajectory_frames(n, seed=2)
    geo = featx_ref.Geometry(30.0 / 512, 512, d["bearings"])
    maps = _lib.Maps(ctx, geo.map_x, geo.map_y, 512, 512, geo.width, geo.height)
    return d["frames"].numpy(), d["poses_odom"], maps, (lambda: pipeline.FrontEnd(ctx, maps, max_frames=n, **kw))


@pytest.mark.parametrize("mode", ["cold", "carry", "plane"])
def test_run_jpeg_host_equals_run_host_on_cv2_frames(gpu_ctx, mode):
    from sonar_slam_b200 import _lib
    kw = dict(min_points=30)
    if mode == "plane":
        kw["icp"] = _lib.IcpParams(minimizer=1, normals_knn=5)
    frames, poses, maps, make = _frontend(gpu_ctx, 40, **kw)
    streams = [jpeg_ref.encode(f, q, s) for f, q, s in zip(frames, itertools.cycle((80, 95, 50)),
                                                            itertools.cycle(("gray", "gray", "420")))]
    decoded = np.stack([jpeg_ref.cv2_gray(b) for b in streams])
    keys = ("T", "iterations", "inliers", "status", "npoints")
    for chunk in (7, 16, 256):
        a, b = make(), make()
        if mode == "carry":
            a.set_carry(True), b.set_carry(True)
            ra = [a.run_host(decoded[s], poses[s], chunk_frames=chunk) for s in (slice(0, 25), slice(25, 40))]
            rb = [b.run_jpeg_host(streams[s], poses[s], chunk_frames=chunk) for s in (slice(0, 25), slice(25, 40))]
        else:
            ra, rb = [a.run_host(decoded, poses, chunk_frames=chunk)], [b.run_jpeg_host(streams, poses, chunk)]
        for x, y in zip(ra, rb):
            for k in keys:
                assert np.array_equal(x[k], y[k]), (mode, chunk, k)
        assert (ra[0]["status"] == 0).sum() > 10


def test_run_jpeg_host_names_the_first_bad_frame(gpu_ctx):
    from sonar_slam_b200 import _lib
    frames, poses, maps, make = _frontend(gpu_ctx, 6)
    streams = [jpeg_ref.encode(f, 80) for f in frames]
    fe = make()
    with pytest.raises(_lib.SonarFEError, match="frame 3: progressive"):
        fe.run_jpeg_host(streams[:3] + [cv2.imencode(".jpg", frames[3], [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()]
                         + streams[4:], poses)
    with pytest.raises(_lib.SonarFEError, match="frame 4: corrupt"):
        fe.run_jpeg_host(streams[:4] + [streams[4][:len(streams[4]) // 2]] + streams[5:], poses, chunk_frames=2)
    assert (fe.run_jpeg_host(streams, poses)["status"] >= 0).all()


def test_feature_extraction_decode_on_device(gpu_ctx):
    import types
    from sonar_slam_b200.bruce_slam.feature_extraction import FeatureExtraction
    fe = FeatureExtraction()
    fe.init_node({"CFAR": {"Ntc": 40, "Ngc": 10, "Pfa": 0.1, "rank": 10, "alg": "SOCA"},
                  "filter": {"threshold": 65, "resolution": 0.5, "radius": 1.0, "min_points": 5, "skip": 1},
                  "compressed_images": True})
    img = synth.make_frame(3)
    full = jpeg_ref.encode(img, 80)
    for b in (full, jpeg_ref.encode(img, 90, "420", True, 5), cv2.imencode(".png", img)[1].tobytes(),
              cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes(),
              full[:len(full) * 3 // 4]):                               # truncated: the device refuses, cv2 decides
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
    ping = synth.Ping(ping_id=0, image=types.SimpleNamespace(data=jpeg_ref.encode(img, 80)), range_resolution=30.0 / 512,
                      num_ranges=512, bearings=synth.bearings_uniform(512))
    fe.decode_on_device = False
    want = fe.callback(ping).copy()
    fe.decode_on_device = True
    assert np.array_equal(fe.callback(ping), want)


def test_header_variants_decode_like_cv2(gpu_ctx):
    cases = [(n, b) for n, (b, st) in jpeg_ref.header_variants().items() if st == "OK"]
    out, st = jpeg.decode_host([b for _, b in cases], 64, 48, ctx=gpu_ctx)
    for i, (name, b) in enumerate(cases):
        assert st[i] == jpeg.OK and np.array_equal(out[i], jpeg_ref.cv2_gray(b)), name


def test_over_long_and_truncated_streams_among_valid_frames(gpu_ctx):
    """Data past the last MCU (an over-long stream, SOF height lowered) is skipped as libjpeg-turbo skips it: the frame
    equals cv2.  A stream that ends early is CORRUPT.  The valid frames of the same call, decoded concurrently, stay
    bit-identical to cv2 -- the over-long frame writes nothing past its own blocks."""
    frames = synth.make_frames(range(4))
    tall = np.concatenate([synth.make_frame(9), np.zeros((512, 512), np.uint8)])
    over = [jpeg_ref.with_sof_size(jpeg_ref.encode(np.zeros((1024, 512), np.uint8), 80), 512),
            jpeg_ref.with_sof_size(jpeg_ref.encode(tall, 95, "420", True, 7), 512)]
    good = [jpeg_ref.encode(f, 80, s, False, r) for f, s, r in zip(frames, ("gray", "420", "444", "gray"), (0, 3, 0, 1))]
    ecs = jpeg_ref.parse(good[0])["ecs"]
    short = good[0][:ecs + (len(good[0]) - ecs) * 2 // 3]
    batch = [over[0], good[0], over[1], good[1], short, good[2], over[0], good[3], over[0]]
    out, st = jpeg.decode_host(batch, 512, 512, ctx=gpu_ctx)
    assert st.tolist() == [jpeg.OK] * 4 + [jpeg.CORRUPT] + [jpeg.OK] * 4
    for i, b in enumerate(batch):
        if i != 4:
            assert np.array_equal(out[i], jpeg_ref.cv2_gray(b)), i
    assert not out[4].any()
    one, s1 = jpeg.decode_host([over[0]], 512, 512, ctx=gpu_ctx)   # alone: the last frame of its call
    assert s1[0] == jpeg.OK and np.array_equal(one[0], out[0])


def test_stage_timing(gpu_ctx):
    streams = [jpeg_ref.encode(f, 80) for f in synth.make_frames(range(4))]
    jpeg.set_timing(True, ctx=gpu_ctx)
    jpeg.decode_host(streams, 512, 512, ctx=gpu_ctx)
    t = jpeg.get_timing(ctx=gpu_ctx)
    jpeg.set_timing(False, ctx=gpu_ctx)
    assert list(t) == list(jpeg.STAGES) and all(ms > 0 and calls == 1 for ms, calls in t.values())
