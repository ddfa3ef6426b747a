"""The ABI of the KNN index's plane budget (hrag_knn_set_memory / hrag_knn_planes_info) and the drop-in's
knn_device_bytes option, without a GPU: the exported symbols, the ctypes signatures against the header, and the
argument checks of accelerate."""
import ctypes as C
import os
import re

import pytest

from hipporag_b200 import _lib
from tests import fake_hipporag

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ("hrag_knn_set_memory", "hrag_knn_planes_info")


def _prototypes():
    text = open(os.path.join(ROOT, "include", "hrag_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return {m.group(1): [a.strip() for a in m.group(2).split(",")]
            for m in re.finditer(r"\bint\s+(hrag_knn_\w+)\s*\(([^)]*)\)\s*;", text)}


@pytest.mark.parametrize("name", ENTRIES)
def test_exported(name):
    lib = C.CDLL(os.path.join(ROOT, "hipporag_b200", "libhrag_b200.so"))
    assert hasattr(lib, name), f"{name} is not exported by libhrag_b200.so"


@pytest.mark.parametrize("name", ENTRIES)
def test_signature_matches_header(name):
    protos = _prototypes()
    assert name in protos, f"{name} is not declared in include/hrag_b200.h"
    res, args = _lib.SIGNATURES[name]
    assert res is C.c_int
    params = protos[name]
    assert len(args) == len(params), f"{name}: {len(args)} ctypes arguments, {len(params)} in the header"
    for ct, p in zip(args, params):
        if "*" in p:
            assert ct is C.c_void_p or issubclass(ct, C._Pointer), f"{name}: {p} is a pointer"
        else:
            assert ct is C.c_int64 and p.startswith("int64_t"), f"{name}: {p} vs {ct}"


def test_planes_info_reports_like_the_fact_planes():
    assert _lib.SIGNATURES["hrag_knn_planes_info"][1] == _lib.SIGNATURES["hrag_fact_planes_info"][1]
    _, args = _lib.SIGNATURES["hrag_knn_planes_info"]
    assert [a._type_ for a in args[1:]] == [C.c_int, C.c_int64, C.c_int64, C.c_int64]


class BudgetEngine:
    """Engine double: records the budgets it is given."""

    def __init__(self):
        self.budgets = []

    def set_mutable(self, on=True):
        pass

    def knn_set_memory(self, n):
        self.budgets.append(n)


def _rag():
    fake_hipporag.install_stub_package()
    from tests.test_accelerate_knn_incremental import EntityRag
    return EntityRag()


def test_accelerate_needs_incremental_for_a_knn_budget():
    import hipporag_b200
    with pytest.raises(ValueError, match="incremental=True"):
        hipporag_b200.accelerate(_rag(), engine=BudgetEngine(), cache=False, knn_device_bytes=1 << 30)


def test_accelerate_rejects_a_negative_knn_budget():
    import hipporag_b200
    with pytest.raises(ValueError, match=">= 0"):
        hipporag_b200.accelerate(_rag(), engine=BudgetEngine(), incremental=True, cache=False, knn_device_bytes=-1)


def test_accelerate_passes_the_budget_before_the_index_is_built(monkeypatch):
    import numpy as np
    import hipporag_b200
    from hipporag_b200 import knn
    eng = BudgetEngine()
    seen = []

    def resident(engine, key_ids, key_vecs, k, thr, prev):
        seen.append(list(engine.budgets))
        return {q: ([q], [1.0]) for q in key_ids}, "built"
    monkeypatch.setattr(knn, "retrieve_knn_resident", resident)
    rag = _rag()
    hipporag_b200.accelerate(rag, engine=eng, incremental=True, cache=False, knn_device_bytes=123456789)
    rag.index((["alpha", "beta"], np.eye(2, 64, dtype=np.float32)))
    assert seen == [[123456789]] and rag._b200_state["last_knn"] == "built"
