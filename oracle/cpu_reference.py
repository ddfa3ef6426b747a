"""CPU baseline that mirrors what the reference actually executes per query, in the
reference's own dtypes -- the timed ``cpu_baseline`` / ``--impl reference`` leg of bench.py.
TEST / BENCH INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

``oracle/retrieve.py`` is the float64 *arbiter*; this file is the *stopwatch*: the same serial
one-query-at-a-time loop as ``HippoRAG.retrieve`` (reference ``src/hipporag/HippoRAG.py:459-480``)
with fp32 BLAS ``np.dot`` for the two similarities (``:1459``, ``:1496``), full ``np.argsort``
(``:1500``, ``:1688``, ``:1746``) and a PPR solve to PRPACK's 1e-10 tolerance.  python-igraph is
not installable offline, so the PPR is a scipy float64 CSR power iteration (kind = "port");
the O(N)/O(P) Python dict loops of ``:1535-1539`` / ``:1629-1635`` are replaced by array
indexing, which only makes this baseline faster than the real reference.
"""
from __future__ import annotations

import time

import numpy as np

from . import ppr as _ppr
from .retrieve import Tables, min_max_normalize, seed_vector


def retrieve_serial(P_csr, tables: Tables, fact_emb: np.ndarray, passage_emb: np.ndarray,
                    Q_fact: np.ndarray, Q_pass: np.ndarray, link_top_k: int = 5,
                    passage_node_weight: float = 0.05, damping: float = 0.5, top_k: int = 200,
                    ppr_tol: float = 1e-10):
    """Returns (ids [Q, top_k], scores [Q, top_k], seconds, per-stage seconds dict)."""
    nq = Q_fact.shape[0]
    ids = np.empty((nq, top_k), dtype=np.int64)
    scores = np.empty((nq, top_k))
    t_sim = t_ppr = t_misc = 0.0
    t_all = time.perf_counter()
    for q in range(nq):
        t0 = time.perf_counter()
        fs = min_max_normalize(np.dot(fact_emb, Q_fact[q]))               # :1459-1461 (fp32 sgemv)
        cand = np.argsort(fs)[-link_top_k:][::-1]                         # :1688
        ps = min_max_normalize(np.dot(passage_emb, Q_pass[q]))            # :1496-1498
        order = np.argsort(ps)[::-1]                                      # :1500
        t1 = time.perf_counter()
        r, _ = seed_vector(tables, fs, list(cand), ps, link_top_k, passage_node_weight)   # :1577-1638
        t2 = time.perf_counter()
        pi = _ppr.ppr_power(P_csr, r, damping, tol=ppr_tol)               # :1736-1743
        doc = pi[tables.passage_vid]                                      # :1745
        o = np.argsort(doc)[::-1][:top_k]                                 # :1746, :503
        t3 = time.perf_counter()
        ids[q, :len(o)] = o
        scores[q, :len(o)] = doc[o]
        t_sim += t1 - t0
        t_misc += t2 - t1
        t_ppr += t3 - t2
        del order
    total = time.perf_counter() - t_all
    return ids, scores, total, dict(sim=t_sim, seeds=t_misc, ppr=t_ppr)


class _RowBlockSpMM:
    """y = A @ X (fp32 CSR x dense) over all host cores: the CSR is cut into row blocks and each block's
    product runs on its own thread (scipy's sparsetools kernels release the GIL); torch's CSR matmul is timed
    against it once and the faster of the two is kept."""

    def __init__(self, A_csr32, threads: int):
        import scipy.sparse as sp
        from concurrent.futures import ThreadPoolExecutor
        self.A = A_csr32
        n = A_csr32.shape[0]
        self.threads = max(1, threads)
        nblk = min(self.threads * 4, max(1, n // 4096))
        cuts = np.linspace(0, n, nblk + 1).astype(np.int64)
        self.blocks = [(int(a), int(b), sp.csr_matrix(A_csr32[int(a):int(b)])) for a, b in zip(cuts[:-1], cuts[1:])]
        self.pool = ThreadPoolExecutor(self.threads)
        self.torch_A = None
        self.use_torch = False

    def _blocks_mm(self, X, out):
        def work(item):
            a, b, blk = item
            out[a:b] = blk @ X
        list(self.pool.map(work, self.blocks))
        return out

    def calibrate(self, X):
        out = np.empty_like(X)
        t0 = time.perf_counter(); self._blocks_mm(X, out); t_blocks = time.perf_counter() - t0
        t_torch = float("inf")
        try:
            import warnings
            import torch
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                A = self.A
                self.torch_A = torch.sparse_csr_tensor(torch.from_numpy(A.indptr.astype(np.int64)),
                                                       torch.from_numpy(A.indices.astype(np.int64)),
                                                       torch.from_numpy(A.data), size=A.shape)
                Xt = torch.from_numpy(X)
                self.torch_A @ Xt
                t0 = time.perf_counter(); self.torch_A @ Xt; t_torch = time.perf_counter() - t0
        except Exception:
            self.torch_A = None
        self.use_torch = t_torch < t_blocks
        return {"row_blocks_threads_s": t_blocks, "torch_csr_s": t_torch}

    def __call__(self, X, out):
        if self.use_torch:
            import torch
            out[:] = (self.torch_A @ torch.from_numpy(X)).numpy()
            return out
        return self._blocks_mm(X, out)


def retrieve_vectorized(P_csr, tables: Tables, fact_emb: np.ndarray, passage_emb: np.ndarray,
                        Q_fact: np.ndarray, Q_pass: np.ndarray, link_top_k: int = 5,
                        passage_node_weight: float = 0.05, damping: float = 0.5, top_k: int = 200,
                        batch: int = 64, sweeps: int = 14, threads: int = 0):
    """BEST-EFFORT CPU implementation of the same path (SURVEY.md 8(d)(2)): not how the reference runs, but what a
    careful numpy/scipy rewrite would do on the host -- so the GPU speed-up is not quoted against a strawman only.
    Batched fp32 sgemm for both similarities (BLAS, all cores), argpartition instead of full argsorts, and a batched
    fp32 CSR SpMM PPR (Chebyshev semi-iteration, the same sweep count as the GPU's fp32 solver) over all cores.
    Returns (ids, scores, seconds, per-stage seconds, info)."""
    import os
    threads = threads or (os.cpu_count() or 1)
    nq = Q_fact.shape[0]
    n = P_csr.shape[0]
    P32 = P_csr.astype(np.float32)
    spmm = _RowBlockSpMM(P32, threads)
    info = spmm.calibrate(np.ones((n, min(batch, nq)), dtype=np.float32))
    pv = np.asarray(tables.passage_vid)
    ids = np.empty((nq, top_k), dtype=np.int64)
    scores = np.empty((nq, top_k), dtype=np.float32)
    t_sim = t_ppr = t_misc = 0.0
    t_all = time.perf_counter()
    for q0 in range(0, nq, batch):
        qs = slice(q0, min(nq, q0 + batch))
        nb = qs.stop - qs.start
        t0 = time.perf_counter()
        Sf = Q_fact[qs] @ fact_emb.T                                        # [nb, F] sgemm
        mn, mx = Sf.min(axis=1, keepdims=True), Sf.max(axis=1, keepdims=True)
        cand = np.argpartition(Sf, -link_top_k, axis=1)[:, -link_top_k:]
        cs = np.take_along_axis(Sf, cand, axis=1)
        o = np.argsort(-cs, axis=1, kind="stable")
        cand, cs = np.take_along_axis(cand, o, axis=1), np.take_along_axis(cs, o, axis=1)
        rng_f = np.where(mx - mn == 0, 1.0, mx - mn)
        cs = (cs - mn) / rng_f
        Sp = Q_pass[qs] @ passage_emb.T                                     # [nb, P] sgemm
        pmn, pmx = Sp.min(axis=1, keepdims=True), Sp.max(axis=1, keepdims=True)
        Sp = (Sp - pmn) / np.where(pmx - pmn == 0, 1.0, pmx - pmn)
        t1 = time.perf_counter()
        V = np.zeros((n, nb), dtype=np.float32)
        V[pv, :] = (Sp * np.float32(passage_node_weight)).T
        for b in range(nb):                                                 # <= 10 phrase seeds per query
            w: dict = {}
            cnt: dict = {}
            for f, s in zip(cand[b], cs[b]):
                for vtx in (tables.fact_subj_vid[f], tables.fact_obj_vid[f]):
                    if vtx < 0:
                        continue
                    c = tables.ent_chunk_count[vtx]
                    w[vtx] = w.get(vtx, 0.0) + float(s) / (c if c > 0 else 1)
                    cnt[vtx] = cnt.get(vtx, 0) + 1
            top = sorted(((w[k] / cnt[k], -k) for k in w), reverse=True)[:link_top_k]
            for val, negk in top:
                V[-negk, b] += val
        t2 = time.perf_counter()
        # Chebyshev semi-iteration on (I - aP) x = v, spectrum of aP in [-a, a]
        x_prev, x, y = None, V.copy(), np.empty_like(V)
        rho2, wk = damping * damping, 1.0
        for it in range(1, sweeps + 1):
            spmm(x, y)
            y *= np.float32(damping)
            y += V
            if it >= 2:
                wk = 1.0 / (1.0 - rho2 / 2.0) if it == 2 else 1.0 / (1.0 - rho2 * wk / 4.0)
                y *= np.float32(wk)
                y += np.float32(1.0 - wk) * x_prev
            x_prev, x, y = x, y, (x_prev if x_prev is not None and it >= 2 else np.empty_like(V))
        doc = (x[pv, :] / x.sum(axis=0, keepdims=True)).T                   # [nb, P]
        part = np.argpartition(-doc, min(top_k, doc.shape[1] - 1), axis=1)[:, :top_k]
        ps = np.take_along_axis(doc, part, axis=1)
        o = np.argsort(-ps, axis=1, kind="stable")
        t3 = time.perf_counter()
        ids[qs, :part.shape[1]] = np.take_along_axis(part, o, axis=1)
        scores[qs, :part.shape[1]] = np.take_along_axis(ps, o, axis=1)
        t_sim += t1 - t0
        t_misc += t2 - t1
        t_ppr += t3 - t2
    total = time.perf_counter() - t_all
    spmm.pool.shutdown()
    info.update(spmm="torch_csr" if spmm.use_torch else "scipy_row_blocks", threads=threads, batch=batch,
                sweeps=sweeps)
    return ids, scores, total, dict(sim=t_sim, seeds=t_misc, ppr=t_ppr), info
