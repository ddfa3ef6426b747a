"""No-GPU check of the float64 stage B entry point: declared in include/hrag_b200.h, exported by libhrag_b200.so, and
bound in _lib.py with argtypes that match the declaration parameter for parameter."""
import ctypes as C
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CTYPES = {"hrag_t*": C.c_void_p, "int32_t": C.c_int32, "double": C.c_double, "float": C.c_float,
           "const float*": C.c_void_p, "const int32_t*": C.c_void_p, "const uint8_t*": C.c_void_p,
           "int32_t*": C.c_void_p, "double*": C.c_void_p}


def _declaration(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "hrag_b200.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m, f"{name} is not declared in include/hrag_b200.h"
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    return [re.sub(r"\s*\w+$", "", p).replace(" *", "*") for p in params]   # drop the parameter names


def test_stage_b_f64_declared_exported_and_bound():
    from hipporag_b200 import _lib
    types = _declaration("hrag_stage_b_f64")
    assert types == ["hrag_t*", "int32_t", "const float*", "const int32_t*", "const float*", "int32_t",
                     "const uint8_t*", "double", "float", "int32_t", "int32_t", "double", "int32_t*", "double*"]
    lib = _lib.load()
    assert hasattr(lib, "hrag_stage_b_f64")
    res, args = _lib.SIGNATURES["hrag_stage_b_f64"]
    assert res is C.c_int
    assert args == [_CTYPES[t] for t in types]
    assert list(lib.hrag_stage_b_f64.argtypes) == args
