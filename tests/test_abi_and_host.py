"""CPU-only: the C-ABI library loads and exports what include/sonarfe.h declares; host-side
logic of the drop-in classes (no compute calls -- there is no GPU here)."""
import json
import os
import re

import numpy as np
import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(REPO, "include", "sonarfe.h")).read()
    return sorted(set(re.findall(r"SFE_API[^;(]*?\b(sfe_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol_and_its_version():
    from sonar_slam_b200 import _lib
    lib = _lib.load()
    names = _declared_symbols()
    assert len(names) >= 8
    for n in names:
        assert hasattr(lib, n), f"libsonarfe.so does not export {n}"
    assert lib.sfe_version() == 202


def test_no_cpu_fallback_context_creation_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from sonar_slam_b200 import _lib
    with pytest.raises(_lib.SonarFEError):
        _lib.Context(0)


def test_cfar_class_threshold_factors_match_reference(golden_dir):
    from sonar_slam_b200.bruce_slam.CFAR import CFAR
    for g in json.load(open(os.path.join(golden_dir, "cfar_tau.json"))):
        if "raises" in g:
            with pytest.raises(ValueError, match=g["raises"]):
                CFAR(g["Ntc"], g["Ngc"], g["Pfa"], g["rank"])
            continue
        c = CFAR(g["Ntc"], g["Ngc"], g["Pfa"], g["rank"])
        for alg in ("CA", "SOCA", "GOCA", "OS"):
            got = getattr(c, "threshold_factor_" + alg)
            assert got == pytest.approx(g[alg], rel=1e-12, abs=0), (g, alg)
        assert str(c) == g["str"]
        assert c.params["SOCA"][:2] == (g["Ntc"] // 2, g["Ngc"] // 2)
        assert c.params["OS"][2] == (g["rank"] if g["rank"] is not None else g["Ntc"] / 2)


def test_cfar_class_asserts_like_reference():
    from sonar_slam_b200.bruce_slam.CFAR import CFAR
    for bad in [(41, 10, 0.1, 1), (40, 9, 0.1, 1), (40, 10, 0.1, 40), (40, 10, 0.1, -1)]:
        with pytest.raises(AssertionError):
            CFAR(*bad)


def test_cfar_module_argument_checks_happen_before_any_device_work():
    from sonar_slam_b200.bruce_slam import cfar
    img = np.zeros((64, 32), np.uint8)
    with pytest.raises(TypeError):
        cfar.soca(np.zeros((4, 4, 4)), 20, 5, 1.0)      # not 2-D
    with pytest.raises(TypeError):
        cfar.soca(img, 20.0, 5, 1.0)                    # pybind's `int train_hs` rejects floats
    with pytest.raises(TypeError):
        cfar.os(img, 20, 5, 10.0, 1.0)                  # rank=None -> Ntc/2 float (CFAR.py:24) is rejected too
    with pytest.raises(TypeError):
        cfar.ca(np.zeros((4, 4), dtype=complex), 1, 1, 1.0)


def test_compressed_ping_is_decoded_like_the_reference():
    """feature_extraction.py:210-213: cv2.imdecode(..., IMREAD_COLOR) then BGR -> gray; PNG is lossless, so the decoded
    ping equals the raw one; the uncompressed branch passes arrays through."""
    import types
    cv2 = pytest.importorskip("cv2")
    from sonar_slam_b200 import synth
    from sonar_slam_b200.bruce_slam.feature_extraction import FeatureExtraction
    img = synth.make_frame(seed=1)
    ok, png = cv2.imencode(".png", img)
    assert ok
    fe = FeatureExtraction()
    fe.compressed_images = True
    got = fe.ping_image(types.SimpleNamespace(ping=types.SimpleNamespace(data=png.tobytes())))
    want = cv2.cvtColor(np.array(cv2.imdecode(np.frombuffer(png.tobytes(), np.uint8), cv2.IMREAD_COLOR)).astype(np.uint8),
                        cv2.COLOR_BGR2GRAY)
    assert got.dtype == np.uint8 and np.array_equal(got, want) and np.array_equal(got, img)
    with pytest.raises(ValueError):
        fe.ping_image(types.SimpleNamespace(ping=types.SimpleNamespace(data=b"not an image")))
    fe.compressed_images = False
    assert np.array_equal(fe.ping_image(types.SimpleNamespace(ping=img)), img)


# ------------------------------------------------------------------ the ctypes binding against the header, entry by entry
def _header_text():
    text = open(os.path.join(REPO, "include", "sonarfe.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def _kind(decl):
    """'const float *pts' -> 'ptr', 'double tau' -> 'f64', ...  (what a ctypes argtype must be compatible with)"""
    if "*" in decl:
        return "ptr"
    base = decl.replace("const", "").split()
    base = " ".join(base[:-1]) if len(base) > 1 else base[0]       # drop the parameter name
    return {"int": "i32", "int32_t": "i32", "float": "f32", "double": "f64", "uint64_t": "u64", "int64_t": "i64"}[base]


def _ctypes_kind(t):
    import ctypes
    if t is ctypes.c_void_p or t is ctypes.c_char_p or (isinstance(t, type) and issubclass(t, ctypes._Pointer)):
        return "ptr"
    return {ctypes.c_int: "i32", ctypes.c_int32: "i32", ctypes.c_float: "f32", ctypes.c_double: "f64",
            ctypes.c_uint64: "u64", ctypes.c_int64: "i64"}[t]


def test_ctypes_signatures_agree_with_the_header_parameter_by_parameter():
    """Every entry point the Python side types (argtypes) has the header's parameter count and, position by position,
    the header's kind (pointer / int / float / double / 64-bit); a binding that drifted from include/sonarfe.h would
    pass garbage without any error at call time."""
    import ctypes
    from sonar_slam_b200 import _lib
    lib = _lib.load()
    protos = re.findall(r"SFE_API\s+([^;]*?)\b(sfe_[a-z0-9_]+)\s*\(([^;]*?)\)\s*;", _header_text(), flags=re.S)
    assert len(protos) >= 40
    typed = 0
    for ret, name, params in protos:
        fn = getattr(lib, name)
        decls = [" ".join(p.split()) for p in params.split(",")]
        want = [] if decls == ["void"] else [_kind(d) for d in decls]
        if fn.argtypes is not None:
            got = [_ctypes_kind(t) for t in fn.argtypes]
            assert got == want, (name, got, want)
            typed += 1
        else:
            assert want == [], f"{name} takes arguments but has no argtypes"
        ret = " ".join(ret.split())
        if ret == "int":
            assert fn.restype is ctypes.c_int, name
        elif ret == "void":
            assert fn.restype is None, name
        elif ret == "uint64_t":
            assert fn.restype is ctypes.c_uint64, name
        elif ret == "const char *":
            assert fn.restype is ctypes.c_char_p, name
        else:
            raise AssertionError(f"unexpected return type {ret!r} of {name}")
    assert typed >= 38


def _header_struct_fields(name):
    body = re.search(r"typedef struct \{([^}]*)\}\s*" + name + r"\s*;", _header_text(), flags=re.S).group(1)
    fields = []
    for stmt in body.split(";"):
        stmt = " ".join(stmt.split())
        if not stmt:
            continue
        typ, names = stmt.split(" ", 1)
        fields += [(n.strip(), typ) for n in names.split(",")]
    return fields


def test_ctypes_structures_agree_with_the_header_field_by_field():
    import ctypes
    from sonar_slam_b200 import _lib
    from oracle import oracle as orc
    ctype_of = {"int": ctypes.c_int, "float": ctypes.c_float, "double": ctypes.c_double, "sfe_icp_params": _lib.IcpParams}
    for cls, cname in ((_lib.IcpParams, "sfe_icp_params"), (_lib.FrontendParams, "sfe_frontend_params")):
        want = [(n, ctype_of[t]) for n, t in _header_struct_fields(cname)]
        assert [(n, t) for n, t in cls._fields_] == want, cname
    # the oracle's parameter block mirrors the product's (tests hand the same values to both)
    assert [(n, t) for n, t in orc.IcpParams._fields_] == [(n, t) for n, t in _lib.IcpParams._fields_]
    assert ctypes.sizeof(_lib.IcpParams) == 40
