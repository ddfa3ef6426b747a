"""CPU oracle for the HippoRAG online-retrieval hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is part of the product:
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import it, and there only as the checker (or as
the timed CPU baseline), never as the thing shipped.  The product path
(``hipporag_b200``) never imports this package and fails loudly when the CUDA
library is missing.

Parity status
-------------
* Rows A-D, F of SURVEY.md section 8(a) (similarity, min-max, fact top-k, seed
  vector construction, result slicing) are PINNED: ``oracle/ref_harness.py``
  runs the reference's own unmodified ``HippoRAG.index()`` / ``retrieve()``
  offline and ``tests/golden/`` holds its outputs.
* Row E (the PPR solve itself) is **parity unpinned** at the igraph boundary:
  the arithmetic lives in python-igraph 0.11.8 -> igraph C core 0.10.x ->
  PRPACK, none of which is in the reference checkout or installable offline.  The oracle
  restates the published definition (see ``oracle/ppr.py``), is cross-checked
  against ``networkx.pagerank`` (an independent implementation of the same
  definition) and hand-derived closed forms, and a gated test compares with the
  real ``igraph`` whenever it is importable.
"""
