"""CPU: the binding of sfe_icp_source_limit (the largest source the ICP's shared-memory layouts hold; larger ones take
the global-source class) and its argument checks, which run before any device call."""
import ctypes

from sonar_slam_b200 import _lib, ops

SFE_ERR_ARG = -1


def test_binding():
    lib = _lib.load()
    f = lib.sfe_icp_source_limit
    assert f.argtypes == [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    assert callable(ops.icp_source_limit)


def test_dim_outside_2_to_3():
    lib = _lib.load()
    prm = _lib.IcpParams()
    out = ctypes.c_int32(-7)
    for dim in (-1, 0, 1, 4):
        assert lib.sfe_icp_source_limit(None, ctypes.byref(prm), dim, ctypes.byref(out)) == SFE_ERR_ARG
        assert lib.sfe_last_error().decode() == \
            f"sfe_icp_source_limit: points must have 2 or 3 columns (got {dim})"
    assert out.value == -7


def test_null_pointers():
    lib = _lib.load()
    prm = _lib.IcpParams()
    out = ctypes.c_int32(-7)
    for dim in (2, 3):
        for args in ((None, ctypes.byref(prm), dim, ctypes.byref(out)), (None, None, dim, ctypes.byref(out)),
                     (None, ctypes.byref(prm), dim, None)):
            assert lib.sfe_icp_source_limit(*args) == SFE_ERR_ARG
            assert lib.sfe_last_error().decode() == "sfe_icp_source_limit: null pointer"
    assert out.value == -7
