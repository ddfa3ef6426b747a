"""The HRAG_FACT_LO_ON_HOST placement without a GPU: the C declaration and the ctypes signature agree, and the Python
entries reject inconsistent arguments before any device work."""
import ctypes as C
import importlib
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "hrag_b200.h")) as f:
        return f.read()


def test_header_declares_the_placement():
    h = _header()
    assert re.search(r"int hrag_set_fact_placement\(hrag_t\* h, int placement\);", h)
    assert re.search(r"#define HRAG_FACT_PLANES_BY_BUDGET 0\b", h)
    assert re.search(r"#define HRAG_FACT_LO_ON_HOST\s+1\b", h)


def test_signature_matches_header():
    from hipporag_b200 import _lib
    restype, argtypes = _lib.SIGNATURES["hrag_set_fact_placement"]
    assert restype is C.c_int
    assert argtypes == [C.c_void_p, C.c_int]


def test_engine_needs_a_budget_for_lo_on_host():
    import hipporag_b200 as hb
    with pytest.raises(ValueError, match="fact_device_bytes"):
        hb.Engine(0, fact_lo_on_host=True)


def test_accelerate_argument_errors():
    from tests import fake_hipporag
    fake_hipporag.install_stub_package()
    import hipporag_b200
    blob = importlib.import_module("hipporag_b200.accelerate").wrap_share_blob({}, b"engine")
    with pytest.raises(ValueError, match=r"fact_lo_on_host=True\).*fact_device_bytes"):
        hipporag_b200.accelerate(object(), fact_lo_on_host=True)
    with pytest.raises(ValueError, match="fact_lo_on_host"):
        hipporag_b200.accelerate(object(), attach=blob, fact_lo_on_host=True)
    with pytest.raises(ValueError, match="fact_lo_on_host"):
        hipporag_b200.accelerate(object(), attach=blob, fact_device_bytes=1 << 30, fact_lo_on_host=True)
