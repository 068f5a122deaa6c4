"""CPU-only: the packed-cloud and scan-match switches of the front end are declared, bound, and check their arguments
before any device work."""
import ctypes
import os
import re

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_declares_the_switches():
    text = " ".join(open(os.path.join(REPO, "include", "sonarfe.h")).read().split())
    assert ("SFE_API int sfe_frontend_set_clouds(sfe_frontend *fe, float *dst, int64_t capacity_points, "
            "int64_t *offsets, int on_host);") in text
    assert "SFE_API int sfe_frontend_set_scan_match(sfe_frontend *fe, int enable);" in text
    assert re.search(r"SFE_ICP_SKIPPED = 7,[^}]*sfe_frontend_set_scan_match", text)


def test_null_handles_and_arguments_are_refused_without_a_device():
    from sonar_slam_b200 import _lib
    lib = _lib.load()
    assert lib.sfe_frontend_set_clouds.argtypes[2] is ctypes.c_int64
    assert lib.sfe_frontend_set_clouds(None, None, 0, None, 1) == -1
    assert "null handle" in lib.sfe_last_error().decode()
    assert lib.sfe_frontend_set_scan_match(None, 0) == -1
    assert "null handle" in lib.sfe_last_error().decode()
    assert _lib.ERR_CAPACITY == -3 and (_lib.ICP_SKIPPED, _lib.ICP_TOO_LARGE) == (7, 8)
