"""An independent restatement of the ALGORITHM the reference's PPR call runs -- PRPACK's
Gauss-Seidel PageRank -- written from the published method, sharing no code with ``oracle/ppr.py``.
TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

Why it exists: ``oracle/ppr.py`` defines PPR through the linear system ``(I - aP) x = v`` and its
three solvers (LU, power iteration, networkx) all check that one formula.  The reference calls
``graph.personalized_pagerank(..., implementation='prpack')`` (``HippoRAG.py:1736-1743``);
python-igraph 0.11.8 -> igraph C core 0.10 -> bundled PRPACK is not in the reference checkout and is
not installable offline, so the **parity of row E stays unpinned**.  What can be done offline is
to restate what PRPACK computes, from its own formulation, and check that it lands on the same
numbers -- in particular the two claims DESIGN.md makes about the igraph side:

* *sinks restart according to the reset distribution* (igraph >= 0.10 passes ``u = v = reset``
  to PRPACK: the mass of dangling vertices is redistributed by ``u``), and
* *the tolerance is 1e-10* on the undistributed probability mass.

PRPACK's Gauss-Seidel solver (``prpack_solver::solve_via_gs``, as published with the library
and described in the igraph documentation) works on the STOCHASTIC formulation

    x = a * M x + a * (sum of x over dangling vertices) * u + (1 - a) * v ,     sum(x) = 1

where ``M[i, j] = w(j -> i) / outstrength(j)``; it starts from ``x = 0``, sweeps the vertices in
index order updating ``x[i]`` in place from its in-edges (newest values), keeps the dangling
term ``delta`` current inside the sweep, and tracks ``err = 1 - sum(x)`` -- the probability mass
not yet distributed -- with a compensated (Kahan) sum; ``x`` grows monotonically, the sweep loop
ends when ``err < tol`` and the result is L1-normalised.  Self-loops are divided out
(``x_i = (...) / (1 - a * M[i, i])``).  For an undirected igraph graph every edge is an in-edge
of both endpoints; a loop edge counts twice in the strength (igraph's degree convention).

Plain Python loops over an adjacency built from the edge list: meant for graphs of a few
thousand vertices in tests, not for timing.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np


def _in_edges(n: int, src, dst, w) -> Tuple[List[Dict[int, float]], np.ndarray]:
    """Per-vertex dict {neighbour: summed weight} of the undirected multigraph + strengths."""
    adj: List[Dict[int, float]] = [dict() for _ in range(n)]
    strength = np.zeros(n, dtype=np.float64)
    for a, b, x in zip(np.asarray(src).tolist(), np.asarray(dst).tolist(), np.asarray(w, dtype=np.float64).tolist()):
        if not x > 0:            # weight <= 0 (or NaN) carries nothing
            continue
        adj[a][b] = adj[a].get(b, 0.0) + x
        adj[b][a] = adj[b].get(a, 0.0) + x      # for a == b this doubles the diagonal, as igraph counts loops twice
        strength[a] += x
        strength[b] += x
    return adj, strength


def personalized_pagerank_gs(n: int, src, dst, w, reset, damping: float = 0.5, tol: float = 1e-10,
                             max_sweeps: int = 10_000, return_sweeps: bool = False):
    """PRPACK-style Gauss-Seidel PPR of an undirected weighted multigraph; ``u = v = reset``."""
    r = np.asarray(reset, dtype=np.float64)
    r = np.where(np.isnan(r) | (r < 0), 0.0, r)          # run_ppr's sanitisation, HippoRAG.py:1735
    if not r.sum() > 0:
        raise ValueError("reset vector has no positive mass")
    v = r / r.sum()
    u = v
    adj, strength = _in_edges(n, src, dst, w)
    dangling = strength == 0
    a = float(damping)
    x = np.zeros(n, dtype=np.float64)
    delta = 0.0                      # a * (mass currently sitting on dangling vertices)
    err, comp = 1.0, 0.0             # err = 1 - sum(x), Kahan-compensated
    sweeps = 0
    while err >= tol and sweeps < max_sweeps:
        sweeps += 1
        for i in range(n):
            old = x[i]
            acc = 0.0
            self_p = 0.0
            for j, wij in adj[i].items():
                if j == i:
                    self_p = wij / strength[i]
                else:
                    acc += x[j] * (wij / strength[j])
            if dangling[i]:
                # the vertex's own mass comes back through delta * u[i]: solve for x_i with that term excluded
                rest = delta - a * old
                new = (a * acc + rest * u[i] + (1.0 - a) * v[i]) / (1.0 - a * u[i])
                delta = rest + a * new
            else:
                new = (a * acc + delta * u[i] + (1.0 - a) * v[i]) / (1.0 - a * self_p)
            x[i] = new
            # err -= (new - old), compensated
            y = -(new - old) - comp
            t = err + y
            comp = (t - err) - y
            err = t
    out = x / x.sum()
    return (out, sweeps) if return_sweeps else out
