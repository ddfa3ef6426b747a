"""The ABI of the shared index (hrag_index_export / _unexport / _attach / _detach / _share_info) and the drop-in's
share blob, without a GPU: the ctypes signatures against the header, and the blob wrapper's round trip and
rejections."""
import ctypes as C
import importlib
import os
import re

import pytest

from hipporag_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHARE_ENTRIES = ("hrag_index_export", "hrag_index_unexport", "hrag_index_attach", "hrag_index_detach",
                 "hrag_index_share_info")


def _prototypes():
    text = open(os.path.join(ROOT, "include", "hrag_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return {m.group(1): [a.strip() for a in m.group(2).split(",")]
            for m in re.finditer(r"\bint\s+(hrag_index_\w+)\s*\(([^)]*)\)\s*;", text)}


@pytest.mark.parametrize("name", SHARE_ENTRIES)
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


def test_share_info_reports_ints_and_sizes():
    _, args = _lib.SIGNATURES["hrag_index_share_info"]
    assert [a._type_ for a in args[1:]] == [C.c_int, C.c_int64, C.c_int64, C.c_int64]


def test_share_blob_round_trip():
    acc = importlib.import_module("hipporag_b200.accelerate")
    fp = {"format": 1, "n_nodes": 7, "edges_md5": "abc", "fact_keys_md5": "d"}
    engine_blob = bytes(range(256)) * 6
    blob = acc.wrap_share_blob(fp, engine_blob)
    assert blob.startswith(acc.SHARE_MAGIC)
    got_fp, got_blob = acc.unwrap_share_blob(blob)
    assert got_fp == fp and got_blob == engine_blob


def test_share_blob_rejections():
    import json
    import struct
    acc = importlib.import_module("hipporag_b200.accelerate")
    blob = acc.wrap_share_blob({"n_nodes": 1}, b"engine")
    with pytest.raises(ValueError, match="not a blob"):
        acc.unwrap_share_blob(b"x" + blob)
    with pytest.raises(ValueError, match="not a blob"):
        acc.unwrap_share_blob(acc.SHARE_MAGIC[:-1])
    n0 = len(acc.SHARE_MAGIC)
    with pytest.raises(ValueError, match="truncated"):
        acc.unwrap_share_blob(blob[:n0 + 10])
    head = json.dumps({"version": acc.SHARE_VERSION + 1, "fingerprint": {}}).encode()
    with pytest.raises(ValueError, match="version"):
        acc.unwrap_share_blob(acc.SHARE_MAGIC + struct.pack("<I", len(head)) + head + b"engine")


def test_accelerate_attach_excludes_incremental_and_fact_budget():
    from tests import fake_hipporag
    fake_hipporag.install_stub_package()
    import hipporag_b200
    blob = importlib.import_module("hipporag_b200.accelerate").wrap_share_blob({}, b"engine")
    with pytest.raises(ValueError, match="incremental"):
        hipporag_b200.accelerate(object(), attach=blob, incremental=True)
    with pytest.raises(ValueError, match="fact_device_bytes"):
        hipporag_b200.accelerate(object(), attach=blob, fact_device_bytes=1 << 20)
    with pytest.raises(ValueError, match="not a blob"):
        hipporag_b200.accelerate(object(), attach=b"engine")
