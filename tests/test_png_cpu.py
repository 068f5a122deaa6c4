"""CPU: PNG chunk inspection (sfe_png_inspect_host needs no GPU) and the numpy restatement of the decoder
(oracle/png_ref.py) against cv2.imdecode(IMREAD_COLOR) + BGR2GRAY, the reference's own decode
(feature_extraction.py:210-213), and against the stored digests."""
import hashlib
import itertools

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import jpeg_ref, png_ref  # noqa: E402
from sonar_slam_b200 import png, synth  # noqa: E402

SIZES = [(1, 1), (1, 9), (9, 1), (7, 9), (17, 33)]


def _img(h, w, rgb, seed=0):
    img = jpeg_ref.contents(h, w, seed=seed)["synth" if seed % 2 else "noise"]
    return png_ref.rgb_of(img) if rgb else img


def _same(b):
    want = png_ref.cv2_gray(b)
    return want is not None and np.array_equal(png_ref.decode(b), want)


@pytest.mark.parametrize("rgb", [False, True])
def test_oracle_equals_cv2_on_every_filter(rgb):
    for (h, w), f in itertools.product(SIZES, range(5)):
        assert _same(png_ref.write(_img(h, w, rgb, h + w), f)), (h, w, f)
    rng = np.random.default_rng(1)
    for h, w in SIZES:
        assert _same(png_ref.write(_img(h, w, rgb, 3), rng.integers(0, 5, h))), (h, w, "mix")


@pytest.mark.parametrize("strategy", list(png_ref.STRATEGIES))
def test_oracle_equals_cv2_on_every_zlib_option(strategy):
    for level, wbits, idat, rgb in itertools.product((0, 1, 6, 9), (9, 15), (None, 1, -7), (False, True)):
        b = png_ref.write(_img(17, 33, rgb, level), [y % 5 for y in range(17)], level, strategy, wbits, idat)
        assert _same(b), (strategy, level, wbits, idat, rgb)


def test_oracle_equals_cv2_on_cv2_written_pings():
    for seed in range(2):
        img = synth.make_frame(seed)
        for x in (img, png_ref.rgb_of(img)):
            b = cv2.imencode(".png", np.ascontiguousarray(x))[1].tobytes()
            assert _same(b)
    assert np.array_equal(png_ref.cv2_gray(cv2.imencode(".png", img)[1].tobytes()), img)  # lossless


def test_oracle_equals_cv2_on_deflate_edge_cases_and_over_long_data():
    for name, (h, w, b) in png_ref.edge_streams().items():
        assert _same(b), name
        assert png.inspect([b])[0].tolist()[:3] == [png.OK, h, w], name
    img = jpeg_ref.contents(64, 48)["synth"]
    b = png_ref.over_long(img)
    assert np.array_equal(png_ref.cv2_gray(b), img) and np.array_equal(png_ref.decode(b), img)


def test_oracle_reproduces_the_golden_digests(golden_dir):
    g = np.load(f"{golden_dir}/png_streams.npz")
    off = g["offsets"]
    assert len(g["names"]) >= 40 and str(g["cv2_version"]) and "png" in str(g["libpng"]).lower()
    for i, name in enumerate(g["names"]):
        img = png_ref.decode(g["bytes"][off[i]:off[i + 1]].tobytes())
        assert tuple(img.shape) == tuple(g["shapes"][i]), name
        assert hashlib.sha256(img.tobytes()).hexdigest() == g["sha256"][i], name


def test_inspect_reports_the_geometry_of_accepted_streams():
    streams, want = [], []
    for (h, w), rgb, idat in itertools.product(SIZES, (False, True), (None, 1, -7)):
        b = png_ref.write(_img(h, w, rgb), png_ref.SUB, idat=idat)
        streams.append(b)
        want.append((png.OK, h, w, 2 if rgb else 0, sum(1 for t, _, _ in png_ref.chunks(b) if t == b"IDAT")))
    assert [tuple(r) for r in png.inspect(streams)] == want


def test_inspect_rejects_what_the_device_decoder_does_not_take():
    img = jpeg_ref.contents(64, 48)["synth"]
    cases = png_ref.rejected_variants(img)
    cases["jpeg_stream"] = (jpeg_ref.encode(img, 80), "NOT_PNG")
    info = png.inspect([b for b, _ in cases.values()])
    for (name, (b, st)), row in zip(cases.items(), info):
        assert row[0] == getattr(png, st), (name, row, png.status_message(row[0]))
        assert png.status_message(row[0]) != "unknown status"
        if st == "OK":  # accepted variants decode like cv2
            assert _same(b) and np.array_equal(png_ref.cv2_gray(b), img), name
    # the rejected orientation is one imdecode would apply: the decoded image is rotated
    assert png_ref.cv2_gray(cases["exif6"][0]).shape == (48, 64)
    # corrupt streams pass the chunk walk (their failures are found while decoding) and cv2 refuses them
    for name, b in png_ref.corrupt_variants(img).items():
        assert png.inspect([b])[0, 0] == png.OK, name
        assert png_ref.cv2_gray(b) is None, name
