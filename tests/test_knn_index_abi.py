"""No-GPU checks of the resident self-KNN index: its entry points are declared in include/hrag_b200.h, exported by
libhrag_b200.so and bound in _lib.py parameter for parameter; the key-transition classifier of knn.py."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CTYPES = {"hrag_t*": C.c_void_p, "int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "float": C.c_float,
           "const float*": C.c_void_p, "const int64_t*": C.c_void_p, "int32_t*": C.c_void_p, "float*": C.c_void_p,
           "int64_t*": C.c_void_p}
_POINTERS = {"hrag_knn_index_update": {9: C.c_int32}, "hrag_knn_index_info": {1: C.c_int64, 2: C.c_int32, 3: C.c_int32}}

_DECLARED = {
    "hrag_knn_index_update": ["hrag_t*", "int64_t", "int32_t", "const float*", "int", "int64_t", "const int64_t*",
                              "float", "int32_t", "int32_t*"],
    "hrag_knn_index_read": ["hrag_t*", "int64_t", "int64_t", "int32_t*", "float*", "int32_t*"],
    "hrag_knn_index_info": ["hrag_t*", "int64_t*", "int32_t*", "int32_t*"],
    "hrag_knn_index_clear": ["hrag_t*"],
}


def _declaration(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "hrag_b200.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m, f"{name} is not declared in include/hrag_b200.h"
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    return [re.sub(r"\s*\w+$", "", p).replace(" *", "*") for p in params]


def _want(name, types):
    """ctypes of the declared parameters: out-pointers the binding types as POINTER(scalar), the rest void*."""
    out = []
    for i, t in enumerate(types):
        scalar = _POINTERS.get(name, {}).get(i)
        out.append(C.POINTER(scalar) if scalar is not None else _CTYPES[t])
    return [a.__name__ for a in out]


@pytest.mark.parametrize("name", sorted(_DECLARED))
def test_knn_index_entry_declared_exported_and_bound(name):
    from hipporag_b200 import _lib
    types = _declaration(name)
    assert types == _DECLARED[name]
    lib = _lib.load()
    assert hasattr(lib, name)
    res, args = _lib.SIGNATURES[name]
    assert res is C.c_int
    assert [a.__name__ for a in args] == _want(name, types)
    assert [a.__name__ for a in getattr(lib, name).argtypes] == _want(name, types)


def test_classify_keys_survivors_then_appends():
    from hipporag_b200.knn import classify_keys
    old = ["a", "b", "c", "d", "e"]
    assert classify_keys(old, old).tolist() == [0, 1, 2, 3, 4]
    assert classify_keys(old, old + ["f", "g"]).tolist() == [0, 1, 2, 3, 4]
    assert classify_keys(old, ["b", "d"]).tolist() == [1, 3]
    assert classify_keys(old, ["a", "c", "e", "x", "y"]).tolist() == [0, 2, 4]
    assert classify_keys(old, ["x"]).tolist() == []                       # full replacement: nothing kept
    assert classify_keys(old, []).tolist() == []                          # every key deleted
    assert classify_keys([], ["a", "b"]).tolist() == []                   # first keys after an empty list
    assert classify_keys(old, ["a", "b"]).dtype == np.int64


@pytest.mark.parametrize("new", [["b", "a"],                 # reorder
                                 ["a", "c", "b"],            # an old key out of order
                                 ["a", "x", "b"],            # an old key after a new one
                                 ["a", "x", "x"],            # duplicate new keys
                                 ["a", "a"]])                # duplicate kept key
def test_classify_keys_rebuilds(new):
    from hipporag_b200.knn import classify_keys
    assert classify_keys(["a", "b", "c"], new) is None


def test_classify_keys_without_a_valid_old_list():
    from hipporag_b200.knn import classify_keys
    assert classify_keys(None, ["a"]) is None
    assert classify_keys(["a", "a"], ["a"]) is None


def test_resident_exact_thresholds():
    from hipporag_b200.knn import resident_exact
    assert resident_exact(0.8) and resident_exact(0.5) and resident_exact(0.375)
    assert not resident_exact(0.7)                 # float32(0.7) < 0.7
    assert not resident_exact(float("nan"))
