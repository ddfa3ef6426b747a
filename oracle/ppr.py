"""Float64 CPU restatement of the Personalized PageRank the reference delegates to
igraph/PRPACK.  TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

**Parity unpinned at the igraph boundary**: the reference's call site is
reference ``src/hipporag/HippoRAG.py:1736-1743``

    graph.personalized_pagerank(vertices=range(N), damping=damping, directed=False,
                                weights='weight', reset=reset_prob, implementation='prpack')

and the arithmetic is in python-igraph 0.11.8 (``requirements.txt:9``) -> igraph C
core 0.10.x -> bundled PRPACK, which is neither in the reference checkout nor
installed.  What is restated here is the published definition:

* the graph is an undirected multigraph (``config_utils.py:176``); parallel edges
  act as one edge of the summed weight (``HippoRAG.py:907-910`` emits (s,o) and
  (o,s) as two parallel edges); edges with weight <= 0 carry nothing;
* strength ``s_j = sum_i W[i,j]``; ``P[i,j] = W[i,j] / s_j`` (column-stochastic
  where ``s_j > 0``);
* reset distribution ``v = r / sum(r)`` after ``run_ppr``'s own sanitisation
  (NaN / negative -> 0, ``HippoRAG.py:1735``);
* ``pi = x / ||x||_1`` with ``(I - alpha P) x = v`` -- equivalently the fixed
  point of ``x <- alpha P x + (1 - sum(alpha P x)) v``: vertices without
  out-weight ("sinks" = isolated vertices, the graph being undirected) restart
  according to ``v`` (igraph >= 0.10 behaviour; ``dangling='uniform'`` is the
  pre-0.10 behaviour and exists only so a gated test can settle which one a real
  igraph implements).

Three independent solvers are provided so they can check each other:
direct sparse LU, power iteration to 1e-14, and (in tests) ``networkx.pagerank``.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla


def sanitize_reset(reset: np.ndarray) -> np.ndarray:
    """``HippoRAG.py:1735``: NaNs and negatives become zero."""
    reset = np.asarray(reset, dtype=np.float64)
    return np.where(np.isnan(reset) | (reset < 0), 0.0, reset)


def symmetric_weights(n: int, src, dst, w) -> sp.csr_matrix:
    """Summed symmetric weight matrix W of an undirected multigraph edge list.

    Mirrors what the graph built by ``HippoRAG.py:1189-1223`` means to an
    undirected weighted PageRank: every igraph edge (u, v, w) contributes w to
    W[u, v] and W[v, u]; a self-loop contributes twice to the diagonal (it is
    counted twice in the strength, as igraph counts loop edges twice in the
    degree); edges with w <= 0 are dropped.
    """
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    w = np.asarray(w, dtype=np.float64)
    keep = w > 0
    src, dst, w = src[keep], dst[keep], w[keep]
    rows = np.concatenate([src, dst])
    cols = np.concatenate([dst, src])
    vals = np.concatenate([w, w])
    W = sp.coo_matrix((vals, (rows, cols)), shape=(n, n)).tocsr()
    W.sum_duplicates()
    W.sort_indices()
    return W


def transition_matrix(W: sp.csr_matrix):
    """P = W D^-1 (column-normalised), and the strength vector."""
    strength = np.asarray(W.sum(axis=0)).ravel()
    inv = np.zeros_like(strength)
    nz = strength > 0
    inv[nz] = 1.0 / strength[nz]
    P = (W @ sp.diags(inv)).tocsr()
    P.sort_indices()
    return P, strength


def factorize(P: sp.csr_matrix, damping: float = 0.5):
    """Sparse LU of (I - alpha P), reusable across reset vectors."""
    n = P.shape[0]
    return spla.splu((sp.identity(n, format="csc") - damping * P.tocsc()).tocsc())


def ppr_direct(P: sp.csr_matrix, reset: np.ndarray, damping: float = 0.5,
               dangling: str = "reset", lu=None) -> np.ndarray:
    """Direct sparse solve of (I - alpha P') x = v, L1-normalised."""
    n = P.shape[0]
    r = sanitize_reset(reset)
    tot = r.sum()
    if not tot > 0:
        raise ValueError("reset vector has no positive mass")
    v = r / tot
    if lu is None:
        lu = factorize(P, damping)
    if dangling == "reset":
        x = lu.solve(v)
    elif dangling == "uniform":
        # sinks jump uniformly: P' = P + (1/n) 1 d^T ; solve with Sherman-Morrison
        d = (np.asarray(P.sum(axis=0)).ravel() == 0).astype(np.float64)
        a = lu.solve(v)
        b = lu.solve(np.full(n, 1.0 / n))
        coef = damping * (d @ a) / (1.0 - damping * (d @ b))
        x = a + coef * b
    else:
        raise ValueError(dangling)
    x = np.maximum(x, 0.0)
    return x / x.sum()


def ppr_power(P: sp.csr_matrix, reset: np.ndarray, damping: float = 0.5,
              tol: float = 1e-14, max_iter: int = 1000, dangling: str = "reset",
              return_iters: bool = False):
    """Power iteration x <- alpha P x + (1 - sum(alpha P x)) u, with u = v (reset)
    or for ``dangling='uniform'`` the sink mass spread uniformly."""
    n = P.shape[0]
    r = sanitize_reset(reset)
    tot = r.sum()
    if not tot > 0:
        raise ValueError("reset vector has no positive mass")
    v = r / tot
    is_sink = np.asarray(P.sum(axis=0)).ravel() == 0
    x = v.copy()
    it = 0
    for it in range(1, max_iter + 1):
        y = damping * (P @ x)
        if dangling == "reset":
            xn = y + (1.0 - y.sum()) * v
        else:
            sink_mass = damping * x[is_sink].sum()
            xn = y + (1.0 - damping) * v + sink_mass / n
        err = np.abs(xn - x).sum()
        x = xn
        if err < tol:
            break
    x = x / x.sum()
    return (x, it) if return_iters else x


def personalized_pagerank(n: int, src, dst, w, reset, damping: float = 0.5,
                          method: str = "auto", dangling: str = "reset") -> np.ndarray:
    """Drop-in for the numeric content of ``Graph.personalized_pagerank`` as used at
    ``HippoRAG.py:1736-1743`` (all vertices, undirected, weighted)."""
    P, _ = transition_matrix(symmetric_weights(n, src, dst, w))
    if method == "auto":
        method = "direct" if n <= 200_000 else "power"
    if method == "direct":
        return ppr_direct(P, reset, damping, dangling)
    return ppr_power(P, reset, damping, dangling=dangling)


def ppr_batch_power(P: sp.csr_matrix, R: np.ndarray, damping: float = 0.5,
                    tol: float = 1e-14, max_iter: int = 1000) -> np.ndarray:
    """Batched float64 power iteration; R is [N, B] (columns = queries)."""
    R = sanitize_reset(R)
    V = R / R.sum(axis=0, keepdims=True)
    X = V.copy()
    for _ in range(max_iter):
        Y = damping * (P @ X)
        Xn = Y + (1.0 - Y.sum(axis=0, keepdims=True)) * V
        err = np.abs(Xn - X).sum(axis=0).max()
        X = Xn
        if err < tol:
            break
    return X / X.sum(axis=0, keepdims=True)
