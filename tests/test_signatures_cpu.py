"""CPU: every function include/rf_b200.h declares has the ctypes signature its prototype gives.  Without one, ctypes passes a Python
int as a C int, so a pointer passed that way would be truncated."""
import ctypes as C
import os
import re

from conftest import ROOT

SCALARS = {"int": C.c_int, "unsigned": C.c_uint, "float": C.c_float, "double": C.c_double, "size_t": C.c_size_t}
RESTYPES = {"int": C.c_int, "double": C.c_double, "void": None, "void*": C.c_void_p, "uint8_t*": C.c_void_p, "char*": C.c_char_p}

# These entry points are checked parameter by parameter: structures by their ctypes class, input arrays as typed pointers, every other
# pointer (output arrays, buffers) as a plain address.
EXACT = ("rf_detect_tiled_align", "rf_detect_yuv_tiled_align", "rf_detect_tiled_device", "rf_detect_yuv_tiled_device",
         "rf_detect_oriented_batch", "rf_detect_yuv_oriented_device", "rf_preprocess_oriented", "rf_preprocess_yuv_oriented",
         "rf_detect_views_oriented", "rf_jpeg_exif_orientation")


def _exact_types():
    from retinaface_b200 import capi
    return {"rf_handle": C.c_void_p, "int": C.c_int, "float": C.c_float, "size_t": C.c_size_t,
            "const uint8_t*const*": C.POINTER(C.c_void_p), "const int*": C.POINTER(C.c_int), "const rf_tiling*": C.POINTER(capi.Tiling),
            "const rf_align_params*": C.POINTER(capi.AlignParams), "const rf_yuv_frame*": C.POINTER(capi.YuvFrame),
            "const rf_det**": C.POINTER(C.c_void_p), "const int32_t**": C.POINTER(C.c_void_p),
            "const rf_oriented_view*": C.POINTER(capi._OrientedView),
            "int*out_count": C.POINTER(C.c_int)}          # rf_detect_views_oriented's count: a ctypes int by reference


def _prototypes():
    """{name: (return type, [parameter, ...])} of every function the header declares, comments stripped and whitespace normalised;
    and the names of its pointer typedefs (the handles)."""
    text = open(os.path.join(ROOT, "include", "rf_b200.h")).read()
    text = re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", "", text, flags=re.S))
    handles = set(re.findall(r"typedef\s+struct\s+\w+\s*\*\s*(\w+)\s*;", text))
    protos = {}
    for ret, name, params in re.findall(r"^([\w \t*]*?)\b(rf_\w+)\s*\(([^;]*)\)\s*;", text, re.M):
        assert name not in protos, name
        params = [re.sub(r"\s+", " ", p.strip()) for p in params.split(",")]
        protos[name] = (ret, [] if params == ["void"] else params)
    return protos, handles


def _squash(t):
    """A C type with its spaces dropped around '*': "const int *" -> "const int*"."""
    return re.sub(r"\s*\*\s*", "*", t.strip())


def _is_pointer(t):
    return t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer)


def test_every_export_has_its_prototypes_signature(built_lib):
    from retinaface_b200 import capi
    protos, handles = _prototypes()
    assert sorted(protos) == sorted(capi.EXPORTS)
    lib, raw, exact = capi.load_library(), C.CDLL(built_lib), _exact_types()
    for name in capi.EXPORTS:
        assert hasattr(raw, name), name
        ret, params = protos[name]
        fn = getattr(lib, name)
        assert fn.restype is RESTYPES[_squash(re.sub(r"\bconst\b", "", ret))], (name, ret, fn.restype)
        assert fn.argtypes is not None and len(fn.argtypes) == len(params), (name, fn.argtypes, params)
        for p, got in zip(params, fn.argtypes):
            words = re.sub(r"\bconst\b", "", p).split()
            if "*" in p or "[" in p or words[0] in handles:
                assert _is_pointer(got), (name, p, got)
            else:
                assert len(words) == 2 and words[0] in SCALARS, (name, p)
                assert got is SCALARS[words[0]], (name, p, got)
        if name in EXACT:
            for p, got in zip(params, fn.argtypes):
                t = _squash(re.sub(r"\s*\w+$", "", p))              # the type without the parameter name
                want = exact.get(_squash(p), exact.get(t, C.c_void_p))
                assert t in exact or t.endswith("*"), (name, p)
                assert got == want, (name, p, got, want)
