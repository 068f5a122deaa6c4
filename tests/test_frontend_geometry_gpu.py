"""A bag whose sonar geometry changes (range setting: num_ranges, range resolution, beam count), fed to one batched
front end as one sequence (sfe_frontend_add_geometry + the *_geometry run flavours).  The keyframe clouds are metric,
so the first frames after a change are matched against the keyframes before it, as in the reference's window
(slam.py:632-633).  Every flavour and schedule must equal the per-frame oracle chain bit for bit."""
import cv2
import numpy as np
import pytest
import torch

from oracle import featx_ref, oracle as orc, pipeline_ref
from sonar_slam_b200 import _lib, feature_image, pipeline, synth

pytestmark = pytest.mark.gpu

N, SEED, WINDOW, CHUNK = 40, 21, 3, 8
# (num_ranges, num_beams, max_range): geometry 0 is the creation geometry and sizes the slots
SHAPES = [(512, 512, 30.0), (384, 512, 20.0), (512, 256, 30.0)]
# switches at 13 (inside the run_host chunk [8, 16)), 23 (one frame before 24, a window-deep and chunk boundary), 30
# and 31 (a one-frame run)
GEOMETRY = np.array([0] * 13 + [1] * 10 + [2] * 7 + [1] + [0] * 9, np.int32)
SWITCHES = [13, 23, 30, 31]
assert len(GEOMETRY) == N


@pytest.fixture(scope="module")
def bag(gpu_ctx):
    """The same walls and poses rendered under every geometry, spliced by GEOMETRY."""
    geos, maps, rendered = [], [], []
    for R, B, rmax in SHAPES:
        d = synth.make_trajectory_frames(N, seed=SEED, num_ranges=R, num_beams=B, max_range=rmax)
        geo = featx_ref.Geometry(rmax / R, R, d["bearings"])
        geos.append(geo)
        maps.append(_lib.Maps(gpu_ctx, geo.map_x, geo.map_y, R, B, geo.width, geo.height))
        rendered.append(d["frames"].numpy())
        poses = d["poses_odom"]
    frames = [rendered[g][i] for i, g in enumerate(GEOMETRY)]
    return dict(geos=geos, maps=maps, frames=frames, poses=poses)


def _front_end(ctx, bag, max_frames=N, **kw):
    fe = pipeline.FrontEnd(ctx, bag["maps"][0], max_frames=max_frames, min_points=30, **kw)
    assert [fe.add_geometry(m) for m in bag["maps"][1:]] == [1, 2]
    return fe


def _slots(frames):
    """Device frames for run_dev_geometry: frame i in the first R_g * B_g bytes of its 512 * 512 slot."""
    slots = np.zeros((len(frames), 512 * 512), np.uint8)
    for i, f in enumerate(frames):
        slots[i, :f.size] = f.reshape(-1)
    return torch.from_numpy(slots).cuda()


def _device_results(ctx, fe, n):
    r = fe.results_dev()
    out = {"T": ctx.to_host(r["T"], (n, 3, 3), np.float32)}
    for k in ("iterations", "inliers", "status"):
        out[k] = ctx.to_host(r[k], (n,), np.int32)
    out["npoints"] = ctx.to_host(r["cloud_count"], (n,), np.int32)
    xy = ctx.to_host(r["cloud_xy"], (n, r["cloud_stride"], 2), np.float32)
    out["clouds"] = [xy[i, :c].copy() for i, c in enumerate(out["npoints"])]
    return out


def _host_results(ctx, fe, got):
    n = len(got["status"])
    out = {k: got[k].copy() for k in ("T", "iterations", "inliers", "status", "npoints")}
    out["clouds"] = _device_results(ctx, fe, n)["clouds"]
    return out


def _assert_same(a, b, what):
    assert np.array_equal(a["T"].view(np.uint32), b["T"].view(np.uint32)), what
    for k in ("iterations", "inliers", "status", "npoints"):
        assert np.array_equal(a[k], b[k]), (what, k)
    for i, (x, y) in enumerate(zip(a["clouds"], b["clouds"])):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), (what, "cloud", i)


def _oracle(bag, frames=None):
    """pipeline_ref.run's window / submap / ICP loop over clouds from each frame's own geometry."""
    frames = bag["frames"] if frames is None else frames
    poses, prm = bag["poses"], orc.IcpParams()
    clouds = [pipeline_ref.slam_cloud(pipeline_ref.frame_cloud(f, bag["geos"][g])) for f, g in zip(frames, GEOMETRY)]
    results = []
    for i in range(len(frames)):
        guess = pipeline_ref.between(poses[i - 1], poses[i]) if i > 0 else np.eye(3, dtype=np.float32)
        parts = [pipeline_ref.transform_points(clouds[k], pipeline_ref.between(poses[i - 1], poses[k]))
                 for k in range(max(0, i - WINDOW), i)]
        tgt = np.concatenate(parts) if parts else np.zeros((0, 2), np.float32)
        if len(tgt):
            tgt, _ = orc.downsample(tgt, 0.5)
        if len(clouds[i]) < 30 or len(tgt) < 30:
            results.append(dict(status=7, T=guess, iterations=0, inliers=0))
            continue
        results.append(orc.icp(clouds[i], tgt, guess, prm))
    return clouds, results


@pytest.fixture(scope="module")
def reference(gpu_ctx, bag):
    """run_host_geometry on the spliced bag, checked once against the oracle chain; the other tests compare with it."""
    fe = _front_end(gpu_ctx, bag)
    got = _host_results(gpu_ctx, fe, fe.run_host(bag["frames"], bag["poses"], chunk_frames=CHUNK, geometry=GEOMETRY))
    clouds, want = _oracle(bag)
    for i in range(N):
        assert np.array_equal(got["clouds"][i], clouds[i]), i
        assert got["status"][i] == want[i]["status"], (i, got["status"][i], want[i]["status"])
        if want[i]["status"] == 0:
            assert np.array_equal(got["T"][i].view(np.uint32), want[i]["T"].view(np.uint32)), i
            assert got["iterations"][i] == want[i]["iterations"] and got["inliers"][i] == want[i]["inliers"], i
        else:
            assert np.allclose(got["T"][i], want[i]["T"]), i      # failed / skipped: the guess comes back
    assert np.array_equal(got["npoints"], [len(c) for c in clouds])
    # the frames after every switch are matched against the keyframes before it, not skipped
    for s in SWITCHES:
        assert got["status"][s] == 0, (s, got["status"][s])
    assert (got["status"] == 0).sum() >= N - 3
    return got


def test_host_flavour_equals_oracle_chain(reference):
    assert reference["status"][0] == 7


def test_device_flavour(gpu_ctx, bag, reference):
    fe = _front_end(gpu_ctx, bag)
    fe.run_dev(_slots(bag["frames"]).data_ptr(), bag["poses"], N, geometry=GEOMETRY)
    _assert_same(_device_results(gpu_ctx, fe, N), reference, "run_dev")


@pytest.mark.parametrize("chunk", [1, 5, 64])
def test_host_flavour_any_chunk_and_packed_form(gpu_ctx, bag, reference, chunk):
    fe = _front_end(gpu_ctx, bag)
    packed = fe.pack_frames(bag["frames"], GEOMETRY)
    got = fe.run_host(packed, bag["poses"], chunk_frames=chunk, geometry=GEOMETRY)
    _assert_same(_host_results(gpu_ctx, fe, got), reference, ("run_host", chunk))


def test_carry_across_pieces_at_the_switches(gpu_ctx, bag, reference):
    """Pieces whose boundaries fall on and next to the switches, host and device flavours in turn."""
    fe = _front_end(gpu_ctx, bag)
    fe.set_carry(True)
    cuts = [0, 13, 14, 22, 23, 24, 30, 31, 32, N]
    for j, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        if j % 2 == 0:
            got = _host_results(gpu_ctx, fe, fe.run_host(bag["frames"][a:b], bag["poses"][a:b], chunk_frames=4,
                                                         geometry=GEOMETRY[a:b]))
        else:
            slots = _slots(bag["frames"][a:b])
            fe.run_dev(slots.data_ptr(), bag["poses"][a:b], b - a, geometry=GEOMETRY[a:b])
            got = _device_results(gpu_ctx, fe, b - a)
        piece = {k: v[a:b] for k, v in reference.items()}
        _assert_same(got, piece, ("carry", a, b))


def test_compressed_flavours(gpu_ctx, bag, reference):
    fe = _front_end(gpu_ctx, bag)
    png = [cv2.imencode(".png", f)[1].tobytes() for f in bag["frames"]]
    got = fe.run_png_host(png, bag["poses"], chunk_frames=CHUNK, geometry=GEOMETRY)
    _assert_same(_host_results(gpu_ctx, fe, got), reference, "png")
    # JPEG is lossy: the reference is the raw flavour on the frames imdecode gives
    jpg = [cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, 92])[1].tobytes() for f in bag["frames"]]
    decoded = [cv2.cvtColor(cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2GRAY)
               for s in jpg]
    want = _host_results(gpu_ctx, fe, fe.run_host(decoded, bag["poses"], chunk_frames=CHUNK, geometry=GEOMETRY))
    assert (want["status"] == 0).sum() >= N - 4
    got = fe.run_jpeg_host(jpg, bag["poses"], chunk_frames=CHUNK, geometry=GEOMETRY)
    _assert_same(_host_results(gpu_ctx, fe, got), want, "jpeg")
    # a stream that does not decode to its own geometry's shape is named
    with pytest.raises(_lib.SonarFEError, match=r"frame 13 \(geometry 2, 512 x 256\)"):
        fe.run_png_host(png, bag["poses"], geometry=np.where(np.arange(N) == 13, 2, GEOMETRY))


def test_one_geometry_through_the_new_entry_points(gpu_ctx, bag):
    n = 12
    frames, poses = np.stack(bag["frames"][:n]), bag["poses"][:n]
    fe = _front_end(gpu_ctx, bag)
    old = _host_results(gpu_ctx, fe, fe.run_host(frames, poses, chunk_frames=5))
    new = _host_results(gpu_ctx, fe, fe.run_host(frames, poses, chunk_frames=5, geometry=np.zeros(n, np.int32)))
    _assert_same(new, old, "run_host")
    dev = torch.from_numpy(frames).cuda()
    fe.run_dev(dev.data_ptr(), poses, n)
    old = _device_results(gpu_ctx, fe, n)
    fe.run_dev(dev.data_ptr(), poses, n, geometry=np.zeros(n, np.int32))
    _assert_same(_device_results(gpu_ctx, fe, n), old, "run_dev")
    _assert_same(old, new, "run_dev vs run_host")


def test_feature_images_of_a_one_geometry_call(gpu_ctx, bag):
    """All frames in geometry 1: images of that geometry's size, as sfe_feature_image renders them."""
    sel = [i for i, g in enumerate(GEOMETRY) if g == 1][:8]
    frames, poses, m = [bag["frames"][i] for i in sel], bag["poses"][sel], bag["maps"][1]
    want = feature_image.render_host(m, np.stack(frames), ctx=gpu_ctx)
    fe = _front_end(gpu_ctx, bag)
    geometry = np.ones(len(sel), np.int32)
    img = np.zeros((len(sel), m.rows, m.cols, 3), np.uint8)
    plain = fe.run_host(frames, poses, chunk_frames=3, geometry=geometry)
    plain = {k: v.copy() for k, v in plain.items()}
    got = fe.run_host(frames, poses, chunk_frames=3, geometry=geometry, images=img)
    assert np.array_equal(img, want)
    assert np.array_equal(got["T"], plain["T"]) and np.array_equal(got["status"], plain["status"])
    dimg = torch.zeros((len(sel), m.rows, m.cols, 3), dtype=torch.uint8, device="cuda")
    fe.run_dev(_slots(frames).data_ptr(), poses, len(sel), geometry=geometry, images=dimg)
    gpu_ctx.sync()
    assert np.array_equal(dimg.cpu().numpy(), want)


def test_stage_timer_adds_up_the_per_run_launches(gpu_ctx, bag):
    fe = _front_end(gpu_ctx, bag)
    fe.set_timing(True)
    fe.run_dev(_slots(bag["frames"]).data_ptr(), bag["poses"], N, geometry=GEOMETRY)
    t = fe.get_timing()
    runs = 1 + int((np.diff(GEOMETRY) != 0).sum())
    assert t["cfar"][1] == runs and t["cart_points"][1] == runs
    assert t["icp"][1] == 1 and t["cfar"][0] > 0


def test_rejections_before_any_device_work(gpu_ctx, bag):
    fe = _front_end(gpu_ctx, bag)
    small = pipeline.FrontEnd(gpu_ctx, bag["maps"][2], max_frames=4)
    poses, frames = bag["poses"][:4], bag["frames"][:4]
    before = gpu_ctx.launches
    # a geometry larger than the slots
    with pytest.raises(_lib.SonarFEError, match=r"polar shape 512x512 does not fit the front end's 512x256"):
        small.add_geometry(bag["maps"][0])
    # unknown or negative ids, in every flavour
    for bad in (3, -1):
        g = np.array([0, 0, bad, 0], np.int32)
        with pytest.raises(_lib.SonarFEError, match=f"frame 2 has geometry id {bad}"):
            fe.run_host(frames, poses, geometry=g)
        with pytest.raises(_lib.SonarFEError, match=f"frame 2 has geometry id {bad}"):
            fe.run_dev(_slots(frames).data_ptr(), poses, 4, geometry=g)
        with pytest.raises(_lib.SonarFEError, match=f"frame 2 has geometry id {bad}"):
            fe.run_png_host([cv2.imencode(".png", f)[1].tobytes() for f in frames], poses, geometry=g)
    # a frame whose packed size is not its geometry's, and offsets past the end of the packed buffer
    buf, off = fe.pack_frames(frames, GEOMETRY[:4])
    with pytest.raises(_lib.SonarFEError, match="frame 3 has 262144 bytes; its geometry 1 takes 384 x 512"):
        fe.run_host((buf, off), poses, geometry=np.array([0, 0, 0, 1], np.int32))
    with pytest.raises(ValueError, match="overrun the packed buffer"):
        fe.run_host((buf[:-1], off), poses, geometry=GEOMETRY[:4])
    # mixed geometries with feature images
    img = np.zeros((4, bag["maps"][0].rows, bag["maps"][0].cols, 3), np.uint8)
    mixed = np.array([0, 0, 1, 1], np.int32)
    two = [frames[0], frames[1], bag["frames"][13], bag["frames"][14]]
    with pytest.raises(_lib.SonarFEError, match="more than one geometry"):
        fe.run_host(two, poses, geometry=mixed, images=img)
    assert gpu_ctx.launches == before
    # more geometries than the limit
    for _ in range(_lib.MAX_GEOMETRIES - 3):
        fe.add_geometry(bag["maps"][1])
    with pytest.raises(_lib.SonarFEError, match="already has 8 geometries"):
        fe.add_geometry(bag["maps"][1])
    # a rejected call leaves the front end usable
    got = fe.run_host(frames, poses, geometry=np.zeros(4, np.int32))
    assert got["status"][0] == 7 and (got["status"][1:] == 0).all()
