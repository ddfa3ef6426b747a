"""No-GPU check of the index update entry points: declared in include/hrag_b200.h, exported by libhrag_b200.so, and
bound in _lib.py with argtypes that match the declarations parameter for parameter."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CTYPES = {"hrag_t*": C.c_void_p, "int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64,
           "const float*": C.c_void_p, "const int32_t*": C.c_void_p, "const double*": C.c_void_p,
           "void*": C.c_void_p, "int64_t*": C.POINTER(C.c_int64)}

_DECLARED = {
    "hrag_set_mutable": ["hrag_t*", "int"],
    "hrag_index_reserve": ["hrag_t*", "int64_t", "int64_t", "int64_t", "int64_t"],
    "hrag_index_append": ["hrag_t*", "int64_t", "int64_t", "const int32_t*", "const int32_t*", "const double*",
                          "int64_t", "const int32_t*", "int64_t", "const int32_t*", "const int32_t*",
                          "const int32_t*", "int32_t", "const float*", "const float*", "int"],
    "hrag_index_delete": ["hrag_t*", "int64_t", "const int32_t*", "int64_t", "const int32_t*", "const int32_t*"],
    "hrag_debug_index": ["hrag_t*", "int", "void*", "int64_t", "int64_t*"],
}


def _declaration(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "hrag_b200.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m, f"{name} is not declared in include/hrag_b200.h"
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    return [re.sub(r"\s*\w+$", "", p).replace(" *", "*") for p in params]   # drop the parameter names


@pytest.mark.parametrize("name", sorted(_DECLARED))
def test_index_update_entry_declared_exported_and_bound(name):
    from hipporag_b200 import _lib
    types = _declaration(name)
    assert types == _DECLARED[name]
    lib = _lib.load()
    assert hasattr(lib, name)
    res, args = _lib.SIGNATURES[name]
    assert res is C.c_int
    want = [_CTYPES[t] for t in types]
    assert [a.__name__ for a in args] == [a.__name__ for a in want]
    assert [a.__name__ for a in getattr(lib, name).argtypes] == [a.__name__ for a in want]


def test_on_device_bits_match_the_header():
    from hipporag_b200 import _lib
    text = open(os.path.join(ROOT, "include", "hrag_b200.h")).read()
    bits = {k: int(v) for k, v in re.findall(r"#define\s+HRAG_(DEVICE_\w+)\s+(\d+)", text)}
    assert bits == {"DEVICE_EDGES": _lib.DEVICE_EDGES, "DEVICE_FACT_EMB": _lib.DEVICE_FACT_EMB,
                    "DEVICE_PASSAGE_EMB": _lib.DEVICE_PASSAGE_EMB}
