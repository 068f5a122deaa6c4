"""CPU: JPEG header inspection (sfe_jpeg_inspect_host needs no GPU) and the numpy restatement of the decoder
(oracle/jpeg_ref.py) against cv2.imdecode(IMREAD_COLOR) + BGR2GRAY, the reference's own decode
(feature_extraction.py:210-213), and against the stored digests."""
import hashlib
import itertools

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import jpeg_ref  # noqa: E402
from sonar_slam_b200 import jpeg  # noqa: E402

SIZES = [(1, 1), (7, 9), (8, 8), (16, 16), (17, 33)]
GRID = list(itertools.product(SIZES, jpeg_ref.SAMPLINGS, (False, True), (0, 1, 3, 17)))
SAMPLING_CODE = {"gray": jpeg.GRAY, "444": jpeg.S444, "422": jpeg.S422, "420": jpeg.S420}


def test_inspect_reports_the_geometry_of_cv2_streams():
    streams, want = [], []
    for (h, w), samp, opt, ri in GRID:
        streams.append(jpeg_ref.encode(jpeg_ref.contents(h, w)["synth"], 80, samp, opt, ri))
        want.append((jpeg.OK, h, w, 1 if samp == "gray" else 3, SAMPLING_CODE[samp], ri))
    streams.append(jpeg_ref.encode(jpeg_ref.contents(512, 512)["synth"], 80))
    want.append((jpeg.OK, 512, 512, 1, jpeg.GRAY, 0))
    assert [tuple(r) for r in jpeg.inspect(streams)] == want


def _with_exif_orientation(buf, orientation):
    tiff = b"II*\x00" + (8).to_bytes(4, "little") + (1).to_bytes(2, "little") + \
        (0x0112).to_bytes(2, "little") + (3).to_bytes(2, "little") + (1).to_bytes(4, "little") + \
        orientation.to_bytes(2, "little") + b"\x00\x00" + (0).to_bytes(4, "little")
    app1 = b"Exif\x00\x00" + tiff
    return buf[:2] + b"\xff\xe1" + (len(app1) + 2).to_bytes(2, "big") + app1 + buf[2:]


def test_inspect_rejects_what_the_device_decoder_does_not_take():
    img = jpeg_ref.contents(64, 48)["synth"]
    rgb = np.dstack([img, img, img])
    base = jpeg_ref.encode(img, 80)
    cases = {
        "progressive": (cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes(), jpeg.PROGRESSIVE),
        "411": (cv2.imencode(".jpg", rgb, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                           cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411])[1].tobytes(), jpeg.SAMPLING),
        "440": (cv2.imencode(".jpg", rgb, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                           cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440])[1].tobytes(), jpeg.SAMPLING),
        "png": (cv2.imencode(".png", img)[1].tobytes(), jpeg.NOT_JPEG),
        "random": (np.random.default_rng(3).integers(0, 256, 4000, dtype=np.uint8).tobytes(), jpeg.NOT_JPEG),
        "truncated": (base[:100], jpeg.TRUNCATED),
        "empty": (b"", jpeg.NOT_JPEG),
        "exif6": (_with_exif_orientation(base, 6), jpeg.ORIENTATION),
        "exif1": (_with_exif_orientation(base, 1), jpeg.OK),
    }
    info = jpeg.inspect([b for b, _ in cases.values()])
    for (name, (_, st)), row in zip(cases.items(), info):
        assert row[0] == st, (name, row, jpeg.status_message(row[0]))
        if st != jpeg.OK:
            assert row[4] == -1 and jpeg.status_message(row[0]) not in ("ok", "unknown status")
    # the rejected orientation is one imdecode would apply: the decoded image is rotated
    assert jpeg_ref.cv2_gray(cases["exif6"][0]).shape == (48, 64)
    # the 12-bit / arithmetic / lossless / CMYK statuses from hand-edited headers
    sof = base.index(b"\xff\xc0")
    assert jpeg.inspect([base[:sof] + b"\xff\xc9" + base[sof + 2:]])[0, 0] == jpeg.ARITHMETIC
    assert jpeg.inspect([base[:sof] + b"\xff\xc3" + base[sof + 2:]])[0, 0] == jpeg.LOSSLESS
    assert jpeg.inspect([base[:sof + 4] + b"\x0c" + base[sof + 5:]])[0, 0] == jpeg.PRECISION


@pytest.mark.parametrize("samp", jpeg_ref.SAMPLINGS)
def test_oracle_equals_cv2_bit_for_bit(samp):
    n = 0
    for (h, w), s, opt, ri in GRID:
        if s != samp:
            continue
        for name, img in jpeg_ref.contents(h, w, seed=h * 100 + w).items():
            for q in (1, 10, 50, 80, 95, 100):
                b = jpeg_ref.encode(img, q, samp, opt, ri)
                got = jpeg_ref.decode(b)["image"]
                assert np.array_equal(got, jpeg_ref.cv2_gray(b)), ((h, w), name, q, samp, opt, ri)
                n += 1
    assert n == len(SIZES) * 8 * 5 * 6


def test_oracle_reproduces_the_golden_digests(golden_dir):
    g = np.load(f"{golden_dir}/jpeg_streams.npz")
    off = g["offsets"]
    assert len(g["names"]) >= 40 and str(g["cv2_version"]) and "turbo" in str(g["libjpeg"])
    for i, name in enumerate(g["names"]):
        b = g["bytes"][off[i]:off[i + 1]].tobytes()
        img = jpeg_ref.decode(b)["image"]
        assert tuple(img.shape) == tuple(g["shapes"][i]), name
        assert hashlib.sha256(img.tobytes()).hexdigest() == g["sha256"][i], name


def test_header_variants_status_and_oracle():
    """16-bit DQT, Adobe transform 1 and JFIF-less 1/2/3 ids (YCbCr), six distinct Huffman tables are accepted and the
    oracle decodes them like cv2; Adobe transform 0, R/G/B ids and 4 components are rejected as colour spaces."""
    cases = {n: (b, getattr(jpeg, st)) for n, (b, st) in jpeg_ref.header_variants().items()}
    info = jpeg.inspect([b for b, _ in cases.values()])
    for (name, (b, st)), row in zip(cases.items(), info):
        assert row[0] == st, (name, jpeg.status_message(row[0]))
        if st == jpeg.OK:
            assert np.array_equal(jpeg_ref.decode(b)["image"], jpeg_ref.cv2_gray(b)), name
    assert b"\xff\xdb\x00\x83\x10" in cases["dqt16_gray"][0]      # one 16-bit table: 2 + 1 + 128 bytes


def test_trailing_data_after_the_last_mcu_is_skipped_like_libjpeg():
    """An over-long stream (SOF height lowered): libjpeg-turbo decodes the declared rows and skips the rest, and so
    does the oracle; with restart markers, the segments past the last MCU are not read either."""
    img = jpeg_ref.contents(1024, 512)["synth"]
    for ri in (0, 5):
        b = jpeg_ref.with_sof_size(jpeg_ref.encode(img, 80, "gray", False, ri), 512)
        assert jpeg.inspect([b])[0, :3].tolist() == [jpeg.OK, 512, 512]
        assert np.array_equal(jpeg_ref.decode(b)["image"], jpeg_ref.cv2_gray(b))
