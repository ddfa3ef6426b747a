"""CPU checks of the float64 PPR path's host side: the float64 transition CSR, the cache's hi/lo planes, the
fp64-mode prepare of accelerate(), and run_ppr's float64 routing (engine double, no GPU)."""
import os
import tempfile

import numpy as np

from oracle import ppr

NPZ_DEFAULT_KEYS = {"row_ptr", "col", "val", "passage_vid", "fact_subj_vid", "fact_obj_vid", "ent_chunk_count"}


def _edges(seed=0, n=60, m=400):
    rng = np.random.default_rng(seed)
    src, dst = rng.integers(0, n - 3, m), rng.integers(0, n - 3, m)
    w = 10.0 ** rng.uniform(-3, 0, m)          # synonymy-style weights over three decades: not fp32-representable
    w[:20] = rng.integers(1, 4, 20)            # integer weights too (strengths 3, 7, 11, ... appear)
    w[20:30] = -0.5                            # carry nothing
    return n, src, dst, w


def test_transition_csr_float64_equals_oracle():
    from hipporag_b200.engine import build_transition_csr
    n, src, dst, w = _edges()
    row_ptr, col, val = build_transition_csr(n, src, dst, w, dtype=np.float64)
    P, _ = ppr.transition_matrix(ppr.symmetric_weights(n, src, dst, w))
    P.eliminate_zeros()
    assert val.dtype == np.float64
    assert np.array_equal(row_ptr, P.indptr) and np.array_equal(col, P.indices)
    np.testing.assert_array_equal(val, P.data)
    # the default output is unchanged: float32, the rounding of the float64 values
    rp32, col32, val32 = build_transition_csr(n, src, dst, w)
    assert val32.dtype == np.float32
    assert np.array_equal(rp32, row_ptr) and np.array_equal(col32, col)
    np.testing.assert_array_equal(val32, val.astype(np.float32))


def _tables(n):
    return {"passage_vid": np.arange(5, dtype=np.int32), "fact_subj_vid": np.zeros(0, np.int32),
            "fact_obj_vid": np.zeros(0, np.int32), "ent_chunk_count": np.zeros(n, np.int32), "facts": []}


def test_cache_hi_lo_round_trip_reproduces_float64_operator():
    from hipporag_b200 import cache
    from hipporag_b200.engine import build_transition_csr
    n, src, dst, w = _edges(1)
    csr = build_transition_csr(n, src, dst, w, dtype=np.float64)
    fp = {"format": cache.FORMAT_VERSION, "n_nodes": n, "n_facts": 0}
    with tempfile.TemporaryDirectory() as wd:
        cache.save(wd, fp, _tables(n), csr)
        z = np.load(os.path.join(wd, cache.NPZ_NAME))
        assert set(z.files) == NPZ_DEFAULT_KEYS | {"val_lo"}
        assert z["val"].dtype == np.float32 and z["val_lo"].dtype == np.float32
        np.testing.assert_array_equal(z["val"], csr[2].astype(np.float32))
        back = cache.load(wd, fp, fp64=True)
        assert back["val"].dtype == np.float64
        rel = np.abs(back["val"] - csr[2]) / np.abs(csr[2])
        assert rel.max() <= 2.0 ** -45, rel.max()
        assert np.any(back["val"] != back["val"].astype(np.float32))       # the lo plane carries information
        # a default-mode load of the same file sees the fp32 plane only
        np.testing.assert_array_equal(cache.load(wd, fp)["val"], csr[2].astype(np.float32))


def test_default_mode_cache_keys_unchanged():
    from hipporag_b200 import cache
    from hipporag_b200.engine import build_transition_csr
    n, src, dst, w = _edges(2)
    fp = {"format": cache.FORMAT_VERSION, "n_nodes": n, "n_facts": 0}
    with tempfile.TemporaryDirectory() as wd:
        cache.save(wd, fp, _tables(n), build_transition_csr(n, src, dst, w))
        assert set(np.load(os.path.join(wd, cache.NPZ_NAME)).files) == NPZ_DEFAULT_KEYS
        assert cache.load(wd, fp, fp64=True) is None                         # no lo plane: a miss in fp64 mode
        assert cache.load(wd, fp)["val"].dtype == np.float32
    assert cache.FORMAT_VERSION == 1


class RecordingEngine:
    """Engine double: records the CSR it is given and answers ppr / ppr_f64 with the float64 oracle."""
    dim = 0

    def __init__(self):
        self.calls = []

    def load_graph_csr(self, n, row_ptr, col, val):
        import scipy.sparse as sp
        self.n, self.val = n, np.asarray(val)
        self.P = sp.csr_matrix((np.asarray(val, np.float64), col, row_ptr), shape=(n, n))

    def load_tables(self, *a):
        pass

    def load_embeddings(self, fe, pe):
        self.dim = pe.shape[1]

    def set_options(self, **kw):
        pass

    def ppr(self, reset, damping=0.5, iters=0, tol=0.0):
        self.calls.append(("ppr", np.asarray(reset).dtype, tol))
        return ppr.ppr_direct(self.P, reset, damping).astype(np.float32)

    def ppr_f64(self, reset, damping=0.5, tol=0.0):
        self.calls.append(("ppr_f64", np.asarray(reset).dtype, tol))
        return ppr.ppr_direct(self.P, reset, damping)


def _fake_rag(wd):
    from tests import fake_hipporag
    from hipporag_b200 import synth
    fake_hipporag.install_stub_package()
    kg = synth.make_kg(600, 5000, seed=4)
    fe, pe = synth.unit_rows(kg.n_facts, 16, 1), synth.unit_rows(kg.n_pass, 16, 2)
    rag = fake_hipporag.FakeRag(kg, fe, pe, fe[:1], pe[:1], ["q"])
    rag.working_dir = wd
    return rag, kg


def test_fp64_prepare_rewrites_a_default_cache_and_run_ppr_returns_float64():
    import hipporag_b200
    from hipporag_b200 import cache
    with tempfile.TemporaryDirectory() as wd:
        rag, kg = _fake_rag(wd)
        eng = RecordingEngine()
        hipporag_b200.accelerate(rag, engine=eng)
        rag.prepare_retrieval_objects()
        assert eng.val.dtype == np.float32
        assert set(np.load(os.path.join(wd, cache.NPZ_NAME)).files) == NPZ_DEFAULT_KEYS
        # fp64 mode: the default-mode cache lacks val_lo -> miss, float64 upload, cache rewritten with val_lo
        rag64, _ = _fake_rag(wd)
        eng64 = RecordingEngine()
        hipporag_b200.accelerate(rag64, engine=eng64, run_ppr_fp64=True, ppr_tol=1e-12)
        rag64.prepare_retrieval_objects()
        assert rag64._b200_state["cache_hit"] is False
        assert eng64.val.dtype == np.float64
        assert set(np.load(os.path.join(wd, cache.NPZ_NAME)).files) == NPZ_DEFAULT_KEYS | {"val_lo"}
        # the next fp64 prepare hits and uploads P within 2^-45 of what was built
        rag64b, _ = _fake_rag(wd)
        eng64b = RecordingEngine()
        hipporag_b200.accelerate(rag64b, engine=eng64b, run_ppr_fp64=True)
        rag64b.prepare_retrieval_objects()
        assert rag64b._b200_state["cache_hit"] is True and eng64b.val.dtype == np.float64
        np.testing.assert_allclose(eng64b.val, eng64.val, rtol=2.0 ** -45, atol=0)
        # and a default-mode prepare still reads the fp32 plane of the rewritten file
        rag32, _ = _fake_rag(wd)
        eng32 = RecordingEngine()
        hipporag_b200.accelerate(rag32, engine=eng32)
        rag32.prepare_retrieval_objects()
        assert rag32._b200_state["cache_hit"] is True
        np.testing.assert_array_equal(eng32.val, eng64.val.astype(np.float32))
        # run_ppr in fp64 mode: float64 reset and ppr_tol go to ppr_f64; (score desc, index asc) order
        r = np.zeros(kg.n_nodes)
        r[kg.passage_vid[:3]] = [1.0, 1.0, 0.5]
        order, scores = rag64.run_ppr(r, 0.5)
        assert eng64.calls == [("ppr_f64", np.float64, 1e-12)]
        want = ppr.ppr_direct(eng64.P, r, 0.5)[kg.passage_vid]
        assert scores.dtype == np.float64
        assert np.array_equal(order, np.lexsort((np.arange(want.shape[0]), -want)))
        np.testing.assert_array_equal(scores, want[order])
        # default mode keeps the fp32 call
        rag32.run_ppr(r, 0.5)
        assert eng32.calls == [("ppr", np.float32, 0.0)]
