import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # the shared library is a build artefact (git-ignored): build it in-tree when a checkout lacks it
    lib = os.path.join(ROOT, "hipporag_b200", "libhrag_b200.so")
    if not os.path.exists(lib):
        import subprocess
        subprocess.run(["make", "-C", os.path.join(ROOT, "hipporag_b200", "csrc"), "-j8"], check=False,
                       stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device visible")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    """BASELINE config #1 fixture (see tests/golden/make_golden.py) with embeddings rebuilt from seeds."""
    from oracle.ref_harness import seeded_unit_vectors
    from oracle import ppr, retrieve
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "musique1k.npz")))
    dim = int(g["dim"])
    g["fact_emb"] = seeded_unit_vectors(g["fact_seed"], dim)
    g["passage_emb"] = seeded_unit_vectors(g["passage_seed"], dim)
    g["q_fact"] = seeded_unit_vectors(g["qfact_seed"], dim)
    g["q_pass"] = seeded_unit_vectors(g["qpass_seed"], dim)
    n = int(g["n_nodes"])
    W = ppr.symmetric_weights(n, g["edge_src"], g["edge_dst"], g["edge_w"])
    g["P"], g["strength"] = ppr.transition_matrix(W)
    g["tables"] = retrieve.Tables(n, g["passage_vid"], g["fact_subj_vid"], g["fact_obj_vid"],
                                  g["ent_chunk_count"])
    return g
