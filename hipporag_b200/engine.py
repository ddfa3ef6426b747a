"""Python host side of the H100 retrieval engine: thin, typed wrappers over the C ABI.

``Engine`` mirrors the state ``HippoRAG.prepare_retrieval_objects`` materialises
(reference ``src/hipporag/HippoRAG.py:1287-1389``) -- graph, integer tables, fact and
passage embeddings -- as device-resident arrays, and exposes the two GPU stages that bracket the
recognition-memory (LLM) filter of ``HippoRAG.retrieve`` (``:459-480``):

* stage A = ``get_fact_scores`` + the top-k of ``rerank_facts``          (``:1427-1465, 1683-1688``)
* stage B = ``dense_passage_retrieval`` + ``graph_search_with_fact_entities`` + ``run_ppr``
  + the top-k slice of ``_build_retrieval_result``           (``:1467-1502, 1544-1656, 1709-1749, 501-507``)

``B200Retriever`` is the same path on raw arrays (synthetic configs, no HippoRAG object).
Nothing here computes on the CPU: every numeric step is a call into ``libhrag_b200.so``.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import (HragError, PPR_CHEBYSHEV, PPR_FP32, PPR_MIXED, PPR_POWER, SIM_BF16, SIM_BF16X3,  # noqa: F401
                   SIM_FP32)


def build_transition_csr(n_nodes: int, edge_src, edge_dst, edge_w,
                         dtype=np.float32) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """CSR of P = W D^-1 from an igraph-style undirected multigraph edge list.

    Host-side ingest of the graph ``add_new_edges`` builds (``HippoRAG.py:1189-1223``): every
    edge (u, v, w) contributes w to W[u, v] and W[v, u]; parallel edges sum (the reference emits
    each fact as (s, o) and (o, s), ``:907-910``); edges with w <= 0 carry nothing; columns are
    divided by the vertex strength.  Returns (row_ptr int64, col int32, val ``dtype``): float32 by
    default, ``np.float64`` for the operator ``Engine.ppr_f64`` solves with.
    """
    import scipy.sparse as sp
    src = np.asarray(edge_src, dtype=np.int64)
    dst = np.asarray(edge_dst, dtype=np.int64)
    w = np.asarray(edge_w, dtype=np.float64)
    if src.shape != dst.shape or src.shape != w.shape:
        raise ValueError("edge_src, edge_dst, edge_w must have the same length")
    if src.size and (min(src.min(), dst.min()) < 0 or max(src.max(), dst.max()) >= n_nodes):
        raise ValueError("edge endpoint out of range")
    keep = w > 0
    src, dst, w = src[keep], dst[keep], w[keep]
    W = sp.coo_matrix((np.concatenate([w, w]), (np.concatenate([src, dst]), np.concatenate([dst, src]))),
                      shape=(n_nodes, n_nodes)).tocsr()
    W.sum_duplicates()
    W.sort_indices()
    strength = np.asarray(W.sum(axis=0)).ravel()
    inv = np.zeros_like(strength)
    nz = strength > 0
    inv[nz] = 1.0 / strength[nz]
    val = (W.data * inv[W.indices]).astype(dtype)
    return W.indptr.astype(np.int64), W.indices.astype(np.int32), val


def plan_sweeps(damping: float = 0.5, tol: float = 0.0, iters: int = 0, batch: int = 32) -> dict:
    """What the library will run for (damping, tol, iters) on a batch of ``batch`` PPR columns (``hrag_plan_sweeps``;
    pure host code, works without a GPU): solver, sweep counts, predicted relative L1 error."""
    lib = _lib.load()
    mixed, it32, m1, m2 = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    err = C.c_double()
    _lib.check(lib.hrag_plan_sweeps(damping, tol, iters, batch, C.byref(mixed), C.byref(it32), C.byref(m1), C.byref(m2),
                                    C.byref(err)))
    return {"solver": "mixed" if mixed.value else "fp32", "fp32_sweeps": it32.value,
            "mixed_sweeps": (m1.value, 1, m2.value), "predicted_error": err.value}


def shard_rows(n_nodes: int, rank: int, world: int) -> Tuple[int, int]:
    """Node-range partition used by every rank: rows [rank*ceil(N/world), (rank+1)*ceil(N/world))."""
    chunk = -(-n_nodes // world)
    return min(n_nodes, rank * chunk), min(n_nodes, (rank + 1) * chunk)


def balanced_row_bounds(row_ptr, world: int) -> np.ndarray:
    """Work-balanced node-range partition: rank r owns rows [b[r], b[r + 1]) with equal shares of
    cost = non-zeros + 4 per row (a row's epilogue streams cost about four gathers)."""
    row_ptr = np.asarray(row_ptr, dtype=np.int64)
    n = row_ptr.shape[0] - 1
    cost = row_ptr[:-1] + 4 * np.arange(n, dtype=np.int64)          # cost of all rows BEFORE row r
    total = float(row_ptr[-1] + 4 * n)
    b = np.empty(world + 1, dtype=np.int64)
    b[0], b[world] = 0, n
    for k in range(1, world):
        b[k] = int(np.searchsorted(cost, total * k / world, side="left"))
    return np.maximum.accumulate(b)


def slice_csr_rows(row_ptr, col, val, lo: int, hi: int):
    """Rows [lo, hi) of a CSR matrix as a self-contained CSR (columns stay global)."""
    a, b = int(row_ptr[lo]), int(row_ptr[hi])
    return np.ascontiguousarray(row_ptr[lo:hi + 1] - a), col[a:b], val[a:b]


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


def _i32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.int32)


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _stage_b_inputs(q_pass, kept_idx, kept_score, dpr_only):
    """The host arrays of a stage B call: (queries, kept_idx, kept_score (None when no facts), k, dpr flags)."""
    q = _f32(q_pass)
    B = q.shape[0]
    kept_idx, kept_score = _i32(kept_idx), _f32(kept_score)
    kf = kept_idx.shape[1] if kept_idx.ndim == 2 else (kept_idx.size // B if B else 0)
    if kf == 0:
        kept_idx = kept_score = None
    if kf and (kept_idx.size != B * kf or kept_score.size != B * kf):
        raise ValueError("kept_idx / kept_score must be [B, k]")
    flags = None if dpr_only is None else np.ascontiguousarray(dpr_only, dtype=np.uint8)
    return q, kept_idx, kept_score, kf, flags


class Engine:
    """One handle = one H100.  Not thread-safe (like the reference's ``HippoRAG`` object)."""

    def __init__(self, device: int = 0, shard_mode: int = 0, mutable: bool = False, fact_device_bytes: int = 0,
                 fact_lo_on_host: bool = False):
        """``fact_device_bytes`` > 0 caps the device memory of the fact planes (``set_fact_memory``);
        ``fact_lo_on_host`` keeps the hi plane resident and only the lo plane on the host when they exceed it
        (``set_fact_placement``)."""
        if fact_lo_on_host and not fact_device_bytes:
            raise ValueError("Engine(fact_lo_on_host=True) places the fact planes under a device budget: give "
                             "fact_device_bytes > 0 as well")
        self._lib = _lib.load()
        self._h = C.c_void_p()
        dev = (C.c_int * 1)(device)
        _lib.check(self._lib.hrag_create(dev, 1, shard_mode, C.byref(self._h)))
        if mutable:
            self.set_mutable()
        if fact_device_bytes:
            self.set_fact_memory(fact_device_bytes)
        if fact_lo_on_host:
            self.set_fact_placement(True)
        self.device = device
        self.rank, self.world = 0, 1
        self.n_nodes = 0
        self.n_passages = 0
        self.n_facts = 0
        self.dim = 0
        self._keep = []          # device tensors the handle borrows

    # ---------------------------------------------------------------- lifecycle
    def close(self):
        """Free the handle.  Raises ``HragError`` on an owner whose exported index is still attached by other
        processes (their mappings would be left dangling); the handle then stays open."""
        if self._h:
            info = self.share_info()
            if info["role"] == "owner" and info["n_attached"] > 0:
                raise HragError(f"close: {info['n_attached']} handle(s) in other processes are still attached to the "
                                "exported index; they must detach first (the owner must outlive its workers)")
            self._lib.hrag_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---------------------------------------------------------------- multi-GPU
    @staticmethod
    def new_comm_id() -> bytes:
        buf = C.create_string_buffer(128)
        _lib.check(_lib.load().hrag_comm_unique_id(buf))
        return buf.raw

    def init_comm(self, comm_id: bytes, rank: int, world: int):
        buf = C.create_string_buffer(comm_id, 128)
        _lib.check(self._lib.hrag_comm_init(self._h, buf, rank, world))
        self.rank, self.world = rank, world

    def p2p_export(self) -> bytes:
        """64-byte CUDA IPC handle of this rank's PPR state (after init_comm + load_graph)."""
        buf = C.create_string_buffer(64)
        _lib.check(self._lib.hrag_p2p_export(self._h, buf))
        return buf.raw

    def p2p_import(self, handles: Sequence[bytes]):
        """Handles of all ranks in rank order -> fused sweep + exchange (peer stores over NVLink)."""
        blob = C.create_string_buffer(b"".join(handles), 64 * len(handles))
        _lib.check(self._lib.hrag_p2p_import(self._h, blob, len(handles)))

    # ---------------------------------------------------------------- one index shared between processes
    SHARE_ROLES = ("none", "owner", "attached")

    def export_index(self) -> bytes:
        """Export the loaded index to other processes on this GPU (``hrag_index_export``): a blob that
        ``attach`` takes in another process, which then reads this handle's graph, tables and embeddings in place.
        While exported, this handle serves every call as before, but its loads and updates are rejected until
        ``unexport``."""
        n = C.c_int64()
        _lib.check(self._lib.hrag_index_export(self._h, None, 0, C.byref(n)))
        buf = C.create_string_buffer(n.value)
        _lib.check(self._lib.hrag_index_export(self._h, buf, n.value, C.byref(n)))
        return buf.raw[:n.value]

    def unexport(self):
        """End the export (``hrag_index_unexport``); rejected while a handle is attached."""
        _lib.check(self._lib.hrag_index_unexport(self._h))

    def attach(self, blob: bytes):
        """Serve the index another process exported (``export_index``) from this fresh handle, without a copy
        (``hrag_index_attach``).  Loads and updates are rejected until ``detach``."""
        blob = bytes(blob)
        _lib.check(self._lib.hrag_index_attach(self._h, blob, len(blob)))
        self.n_nodes = self.debug_index("ent_chunk_count", size_only=True) // 4
        self.n_passages = self.debug_index("passage_vid", size_only=True) // 4
        self.n_facts = self.debug_index("fact_subj_vid", size_only=True) // 4
        self.dim = 0
        for plane, width, rows in (("passage_hi", 2, self.n_passages), ("passage_f32", 4, self.n_passages),
                                   ("fact_hi", 2, self.n_facts), ("fact_f32", 4, self.n_facts)):
            size = self.debug_index(plane, size_only=True)
            if rows and size:
                self.dim = size // (width * rows)
                break

    def detach(self):
        """Close the mappings of an attached handle (``hrag_index_detach``); it is then an empty handle."""
        _lib.check(self._lib.hrag_index_detach(self._h))
        self.n_nodes = self.n_passages = self.n_facts = self.dim = 0

    def share_info(self) -> dict:
        """``role`` ("none", "owner" or "attached"), ``n_attached`` (live attached handles), ``imported_bytes`` (the
        shared allocations: exported by an owner, mapped by an attached handle) and ``owned_bytes`` (device memory
        this handle allocated itself) (``hrag_index_share_info``)."""
        role, n, imported, owned = C.c_int(), C.c_int64(), C.c_int64(), C.c_int64()
        _lib.check(self._lib.hrag_index_share_info(self._h, C.byref(role), C.byref(n), C.byref(imported),
                                                   C.byref(owned)))
        return {"role": self.SHARE_ROLES[role.value], "n_attached": int(n.value), "imported_bytes": int(imported.value),
                "owned_bytes": int(owned.value)}

    # ---------------------------------------------------------------- uploads
    def set_mutable(self, on: bool = True):
        """Before ``load_graph``: keep the edge list on the device (16 bytes per edge), which ``append`` and
        ``delete`` need (``hrag_set_mutable``)."""
        _lib.check(self._lib.hrag_set_mutable(self._h, 1 if on else 0))

    def set_fact_memory(self, max_device_bytes: int):
        """Before the fact embeddings are loaded: the device bytes their bf16 hi / lo planes (rows x dim x 4 bytes) may
        take (``hrag_set_fact_memory``; 0 = no limit).  A larger fact matrix is kept in pinned host memory and
        streamed through a device ring of at most this many bytes (two slices of a multiple of 256 rows), with
        results bit for bit those of resident planes.  Host planes rule out ``sim_mode=HRAG_SIM_FP32`` for the facts,
        device fact embeddings, ``knn_threshold`` on the facts and in-place updates."""
        _lib.check(self._lib.hrag_set_fact_memory(self._h, int(max_device_bytes)))

    def set_fact_placement(self, lo_on_host: bool):
        """Before the fact embeddings are loaded: where fact planes over the ``set_fact_memory`` budget go
        (``hrag_set_fact_placement``).  ``False`` (the default): both planes in pinned host memory.  ``True``: the hi
        plane stays resident and only the lo plane goes to pinned host memory; stage A then runs the stage-A screen
        on the resident hi plane and reads only the staged candidates' lo rows over PCIe, with results bit for bit
        those of resident planes.  A budget below the hi plane plus two 256-row lo slices fails the load."""
        _lib.check(self._lib.hrag_set_fact_placement(self._h, 1 if lo_on_host else 0))

    def fact_planes_info(self) -> dict:
        """Where the last fact load put the planes: ``on_host`` (0 resident, 1 both planes on the host, 2 the lo
        plane only), the ring's ``slice_rows`` (0 when resident), the planes' ``device_bytes`` (the ring, plus the hi
        plane when only lo is on the host) and the pinned ``host_bytes``."""
        on_host, slice_rows, dev, host = C.c_int(), C.c_int64(), C.c_int64(), C.c_int64()
        _lib.check(self._lib.hrag_fact_planes_info(self._h, C.byref(on_host), C.byref(slice_rows), C.byref(dev),
                                                   C.byref(host)))
        return {"on_host": int(on_host.value), "slice_rows": int(slice_rows.value), "device_bytes": int(dev.value),
                "host_bytes": int(host.value)}

    def _check_device_edges(self, edge_src, edge_dst, edge_w) -> bool:
        """True for three CUDA tensors (checked, and ready to read on the library's stream), False for host arrays."""
        if not any(hasattr(a, "is_cuda") for a in (edge_src, edge_dst, edge_w)):
            return False
        import torch
        want = (torch.int32, torch.int32, torch.float64)
        for a, dt in zip((edge_src, edge_dst, edge_w), want):
            if not (hasattr(a, "is_cuda") and a.is_cuda and a.device.index == self.device and a.dtype == dt
                    and a.dim() == 1 and a.is_contiguous()):
                raise ValueError("a device edge list is three contiguous 1-D CUDA tensors on the handle's device: "
                                 "int32 edge_src, int32 edge_dst, float64 edge_w")
        if not edge_src.shape == edge_dst.shape == edge_w.shape:
            raise ValueError("edge_src, edge_dst, edge_w must have the same length")
        torch.cuda.current_stream(self.device).synchronize()     # the library reads them on its own stream
        return True

    def load_graph(self, n_nodes: int, edge_src, edge_dst, edge_w):
        """igraph-style edge list -> device CSR of P (built by the library on the GPU: hrag_load_graph_coo).

        The edge list may also be three contiguous 1-D CUDA torch tensors on this handle's device -- int32, int32 and
        float64 -- which are read in place (hrag_load_graph_coo_device) and not kept after the call."""
        if self._check_device_edges(edge_src, edge_dst, edge_w):
            _lib.check(self._lib.hrag_load_graph_coo_device(
                self._h, n_nodes, int(edge_src.shape[0]), C.c_void_p(edge_src.data_ptr()),
                C.c_void_p(edge_dst.data_ptr()), C.c_void_p(edge_w.data_ptr())))
            self.n_nodes = n_nodes
            return
        s, d = _i32(edge_src), _i32(edge_dst)
        w = np.ascontiguousarray(edge_w, dtype=np.float64)
        if s.shape != d.shape or s.shape != w.shape:
            raise ValueError("edge_src, edge_dst, edge_w must have the same length")
        _lib.check(self._lib.hrag_load_graph_coo(self._h, n_nodes, int(s.shape[0]), _ptr(s), _ptr(d), _ptr(w)))
        self.n_nodes = n_nodes

    def load_graph_csr(self, n_nodes: int, row_ptr, col, val, balanced: bool = True):
        """Full CSR of P; with node-range sharding this rank's row slice is cut out here -- by default along a
        work-balanced partition (``balanced_row_bounds``), ``balanced=False`` = equal row counts (``shard_rows``).
        A float64 ``val`` also keeps the fp64 operator ``ppr_f64`` needs (``hrag_load_graph_csr_f64``; the fp32
        plane every other solver sweeps is the same ``val.astype(float32)``); any other dtype is loaded as fp32."""
        row_ptr = np.ascontiguousarray(row_ptr, dtype=np.int64)
        f64 = np.asarray(val).dtype == np.float64
        col = _i32(col)
        val = np.ascontiguousarray(val, dtype=np.float64) if f64 else _f32(val)
        lo, hi = (0, n_nodes)
        if self.world > 1:
            if balanced:
                bounds = np.ascontiguousarray(balanced_row_bounds(row_ptr, self.world), dtype=np.int64)
                _lib.check(self._lib.hrag_comm_set_row_bounds(self._h, _ptr(bounds), self.world))
                lo, hi = int(bounds[self.rank]), int(bounds[self.rank + 1])
            else:
                lo, hi = shard_rows(n_nodes, self.rank, self.world)
            row_ptr, col, val = slice_csr_rows(row_ptr, col, val, lo, hi)
        load = self._lib.hrag_load_graph_csr_f64 if f64 else self._lib.hrag_load_graph_csr
        _lib.check(load(self._h, n_nodes, lo, hi, int(col.shape[0]), _ptr(row_ptr), _ptr(col), _ptr(val)))
        self.n_nodes = n_nodes

    def load_tables(self, passage_vid, fact_subj_vid, fact_obj_vid, ent_chunk_count):
        pv, fs, fo, cc = _i32(passage_vid), _i32(fact_subj_vid), _i32(fact_obj_vid), _i32(ent_chunk_count)
        if fs.shape != fo.shape:
            raise ValueError("fact_subj_vid / fact_obj_vid length mismatch")
        if cc.shape[0] != self.n_nodes:
            raise ValueError("ent_chunk_count must have one entry per vertex")
        _lib.check(self._lib.hrag_load_tables(self._h, pv.shape[0], _ptr(pv), fs.shape[0], _ptr(fs), _ptr(fo),
                                              _ptr(cc)))
        self.n_passages, self.n_facts = int(pv.shape[0]), int(fs.shape[0])

    def load_embeddings(self, fact_emb, passage_emb):
        """[F, d] and [P, d] fp32; numpy arrays are copied, CUDA torch tensors are borrowed."""
        for which, emb in ((0, fact_emb), (1, passage_emb)):
            if hasattr(emb, "is_cuda"):      # torch tensor already in HBM
                if not (emb.is_cuda and emb.is_contiguous() and str(emb.dtype) == "torch.float32"):
                    raise ValueError("device embeddings must be contiguous fp32 CUDA tensors")
                rows, dim = (int(emb.shape[0]), int(emb.shape[1])) if emb.dim() == 2 else (0, self.dim or 4)
                _lib.check(self._lib.hrag_load_embeddings(self._h, which, rows, dim, C.c_void_p(emb.data_ptr()), 1))
                self._keep.append(emb)
            else:
                emb = _f32(emb)
                if emb.ndim != 2:
                    emb = emb.reshape(0, self.dim or 4)
                rows, dim = emb.shape
                _lib.check(self._lib.hrag_load_embeddings(self._h, which, rows, dim, _ptr(emb), 0))
            self.dim = dim
            if which == 0:
                self.n_facts = int(rows)
            else:
                self.n_passages = int(rows)

    def load_embeddings_streamed(self, which: int, rows: int, dim: int, chunks):
        """Upload [rows, dim] fp32 embeddings chunk by chunk without ever holding them in fp32 on the device:
        ``chunks`` yields (row0, array) with ``array`` a numpy array or a contiguous fp32 CUDA torch tensor."""
        _lib.check(self._lib.hrag_load_embeddings_begin(self._h, which, rows, dim))
        for row0, emb in chunks:
            if hasattr(emb, "is_cuda"):
                if not (emb.is_cuda and emb.is_contiguous() and str(emb.dtype) == "torch.float32"):
                    raise ValueError("device chunks must be contiguous fp32 CUDA tensors")
                _lib.check(self._lib.hrag_load_embeddings_chunk(self._h, which, int(row0), int(emb.shape[0]),
                                                                C.c_void_p(emb.data_ptr()), 1))
            else:
                emb = _f32(emb)
                _lib.check(self._lib.hrag_load_embeddings_chunk(self._h, which, int(row0), int(emb.shape[0]),
                                                                _ptr(emb), 0))
        self.dim = dim
        if which == 0:
            self.n_facts = int(rows)
        else:
            self.n_passages = int(rows)

    # ---------------------------------------------------------------- incremental updates (mutable handles)
    def reserve(self, nodes: int = 0, edges: int = 0, facts: int = 0, passages: int = 0):
        """Size the capacity of the edge list, tables and embedding planes up front (``hrag_index_reserve``), so no
        later ``append`` copies a plane into a larger allocation."""
        _lib.check(self._lib.hrag_index_reserve(self._h, int(nodes), int(edges), int(facts), int(passages)))

    def _emb_rows(self, emb, name):
        """(pointer, rows, on_device, keep-alive, dim) of new embedding rows: a 2-D numpy array or contiguous fp32
        CUDA tensor on the handle's device."""
        if emb is None:
            return None, 0, False, None, None
        if hasattr(emb, "is_cuda"):
            if not (emb.is_cuda and emb.device.index == self.device and emb.is_contiguous()
                    and str(emb.dtype) == "torch.float32" and emb.dim() == 2):
                raise ValueError(f"device {name} rows must be a contiguous 2-D fp32 CUDA tensor on the handle's device")
            return C.c_void_p(emb.data_ptr()), int(emb.shape[0]), True, emb, int(emb.shape[1])
        a = _f32(emb)
        if a.size == 0:
            return None, 0, False, None, None
        if a.ndim != 2:
            raise ValueError(f"{name} rows must be a 2-D array")
        return _ptr(a), int(a.shape[0]), False, a, int(a.shape[1])

    def _update(self, rc: int):
        """Status of an update entry.  A rejected call leaves the index as it was; one that failed after its inputs
        were checked (out of memory) leaves no index at all, and then the sizes here go to 0 as well."""
        if rc != 0:
            if self.debug_index("ent_chunk_count", size_only=True) == 0:
                self.n_nodes = self.n_passages = self.n_facts = self.dim = 0
            _lib.check(rc)

    def append(self, n_new_nodes: int, edge_src=(), edge_dst=(), edge_w=(), passage_vid=(), fact_subj_vid=(),
               fact_obj_vid=(), ent_chunk_count=None, fact_emb=None, passage_emb=None):
        """``HippoRAG.index()`` on the device (``hrag_index_append``): append ``n_new_nodes`` vertices, the edges (ids
        in the grown range; host arrays or three CUDA tensors as ``load_graph`` takes them), the passage and fact
        rows of the tables with their embedding rows (numpy or CUDA tensors, copied), and replace
        ``ent_chunk_count`` by the whole new table.  The handle then equals a fresh load of the grown arrays."""
        n_new = int(n_new_nodes)
        if self._check_device_edges(edge_src, edge_dst, edge_w):
            ne, es, ed, ew, on_dev = int(edge_src.shape[0]), edge_src, edge_dst, edge_w, _lib.DEVICE_EDGES
            ps, pd, pw = (C.c_void_p(t.data_ptr()) for t in (edge_src, edge_dst, edge_w))
        else:
            es, ed, ew = _i32(edge_src), _i32(edge_dst), np.ascontiguousarray(edge_w, dtype=np.float64)
            if es.shape != ed.shape or es.shape != ew.shape:
                raise ValueError("edge_src, edge_dst, edge_w must have the same length")
            ne, on_dev = int(es.shape[0]), 0
            ps, pd, pw = _ptr(es), _ptr(ed), _ptr(ew)
        pv, fs, fo = _i32(passage_vid), _i32(fact_subj_vid), _i32(fact_obj_vid)
        if fs.shape != fo.shape:
            raise ValueError("fact_subj_vid / fact_obj_vid length mismatch")
        cc = _i32(ent_chunk_count)
        if cc.shape != (self.n_nodes + n_new,):
            raise ValueError("ent_chunk_count must have one entry per vertex of the grown graph")
        fp, f_rows, f_dev, f_keep, f_dim = self._emb_rows(fact_emb, "fact embedding")
        pp, p_rows, p_dev, p_keep, p_dim = self._emb_rows(passage_emb, "passage embedding")
        if f_rows != fs.shape[0] or p_rows != pv.shape[0]:
            raise ValueError("one new embedding row per new fact / passage")
        if f_dim is not None and p_dim is not None and f_dim != p_dim:
            raise ValueError("the new fact and passage rows must share dim")
        dim = f_dim or p_dim or self.dim                    # the library checks it against the index's
        if f_dev or p_dev:
            import torch
            torch.cuda.current_stream(self.device).synchronize()
        on_dev |= (_lib.DEVICE_FACT_EMB if f_dev else 0) | (_lib.DEVICE_PASSAGE_EMB if p_dev else 0)
        self._update(self._lib.hrag_index_append(self._h, n_new, ne, ps, pd, pw, pv.shape[0], _ptr(pv), fs.shape[0],
                                                 _ptr(fs), _ptr(fo), _ptr(cc), dim, fp, pp, on_dev))
        del es, ed, ew, f_keep, p_keep                      # alive until the call has returned
        self.n_nodes += n_new
        self.n_passages += int(pv.shape[0])
        self.n_facts += int(fs.shape[0])

    def delete(self, nodes=(), facts=(), ent_chunk_count=None):
        """``HippoRAG.delete()`` on the device (``hrag_index_delete``): remove the vertices ``nodes`` and the fact rows
        ``facts`` (sorted, unique), renumbering what stays in order; passages whose vertex went are dropped with
        their embedding rows; ``ent_chunk_count`` is the whole new table."""
        nd, fd, cc = _i32(nodes), _i32(facts), _i32(ent_chunk_count)
        if cc.shape != (self.n_nodes - nd.shape[0],):
            raise ValueError("ent_chunk_count must have one entry per remaining vertex")
        self._update(self._lib.hrag_index_delete(self._h, nd.shape[0], _ptr(nd), fd.shape[0], _ptr(fd), _ptr(cc)))
        self.n_nodes -= int(nd.shape[0])
        self.n_facts -= int(fd.shape[0])
        self.n_passages = self.debug_index("passage_vid", size_only=True) // 4

    def set_options(self, ppr_method: Optional[int] = None, ppr_iters: Optional[int] = None,
                    ppr_batch: Optional[int] = None, sim_mode: Optional[int] = None,
                    ppr_precision: Optional[int] = None, mixed_sweeps: Optional[Tuple[int, int]] = None):
        if ppr_precision is not None or mixed_sweeps is not None:
            m1, m2 = mixed_sweeps or (0, 0)
            _lib.check(self._lib.hrag_set_ppr_precision(self._h, -1 if ppr_precision is None else ppr_precision,
                                                        m1, m2))
        _lib.check(self._lib.hrag_set_options(self._h, -1 if ppr_method is None else ppr_method,
                                              -1 if ppr_iters is None else ppr_iters,
                                              -1 if ppr_batch is None else ppr_batch,
                                              -1 if sim_mode is None else sim_mode))

    # ---------------------------------------------------------------- the two GPU stages
    def stage_a(self, q_fact, k: int = 5):
        """-> (top_idx [B,k] int32, top_score [B,k] fp32 min-maxed, n_valid [B] int32)."""
        q = _f32(q_fact)
        B = q.shape[0]
        idx = np.empty((B, k), dtype=np.int32)
        score = np.empty((B, k), dtype=np.float32)
        nv = np.empty(B, dtype=np.int32)
        _lib.check(self._lib.hrag_stage_a(self._h, B, _ptr(q), k, _ptr(idx), _ptr(score), _ptr(nv)))
        return idx, score, nv

    def stage_b(self, q_pass, kept_idx, kept_score, dpr_only=None, damping: float = 0.5,
                passage_node_weight: float = 0.05, link_top_k: int = 5, topk: int = 200,
                iters: int = 0, tol: float = 0.0):
        """-> (ids [B,topk] int32 into passage order, scores [B,topk] fp32), best first.

        ``tol`` = relative L1 accuracy of each PPR vector (0 = 1e-6); the sweep counts follow from
        ``damping`` and ``tol`` unless ``iters`` pins them (``include/hrag_b200.h``)."""
        q, kept_idx, kept_score, kf, flags = _stage_b_inputs(q_pass, kept_idx, kept_score, dpr_only)
        B = q.shape[0]
        ids = np.empty((B, topk), dtype=np.int32)
        scores = np.empty((B, topk), dtype=np.float32)
        _lib.check(self._lib.hrag_stage_b(self._h, B, _ptr(q), _ptr(kept_idx), _ptr(kept_score), kf, _ptr(flags),
                                          damping, passage_node_weight, link_top_k or 0, topk, int(iters),
                                          float(tol), _ptr(ids), _ptr(scores)))
        return ids, scores

    def stage_b_f64(self, q_pass, kept_idx, kept_score, dpr_only=None, damping: float = 0.5,
                    passage_node_weight: float = 0.05, link_top_k: int = 5, topk: int = 200, tol: float = 0.0):
        """``stage_b`` at PRPACK's accuracy (``hrag_stage_b_f64``): the reset in the reference's dtypes, float64 PPR
        with every vector within ``tol`` relative L1 error (0 = 1e-10) by a rigorous bound, float64 gather and exact
        top-k -> (ids [B,topk] int32, scores [B,topk] float64), best first.  Needs a graph loaded from float64 values
        (``load_graph``, or ``load_graph_csr`` with a float64 ``val``)."""
        q, kept_idx, kept_score, kf, flags = _stage_b_inputs(q_pass, kept_idx, kept_score, dpr_only)
        B = q.shape[0]
        ids = np.empty((B, topk), dtype=np.int32)
        scores = np.empty((B, topk), dtype=np.float64)
        _lib.check(self._lib.hrag_stage_b_f64(self._h, B, _ptr(q), _ptr(kept_idx), _ptr(kept_score), kf, _ptr(flags),
                                              float(damping), passage_node_weight, link_top_k or 0, topk, float(tol),
                                              _ptr(ids), _ptr(scores)))
        return ids, scores

    def retrieve_resident(self, d_q_fact, d_q_pass, d_out_ids, d_out_scores, damping: float = 0.5,
                          passage_node_weight: float = 0.05, link_top_k: int = 5, topk: int = 200,
                          iters: int = 0, tol: float = 0.0):
        """Whole path on CUDA torch tensors (identity filter); results land in d_out_*."""
        B = int(d_q_fact.shape[0])
        _lib.check(self._lib.hrag_retrieve_resident(
            self._h, B, C.c_void_p(d_q_fact.data_ptr()), C.c_void_p(d_q_pass.data_ptr()), damping,
            passage_node_weight, link_top_k, topk, int(iters), float(tol), C.c_void_p(d_out_ids.data_ptr()),
            C.c_void_p(d_out_scores.data_ptr())))

    def ppr(self, reset, damping: float = 0.5, iters: int = 0, tol: float = 0.0) -> np.ndarray:
        """``run_ppr``'s numeric core: reset [B, N] (or [N]) -> probabilities, same shape."""
        r = _f32(reset)
        single = r.ndim == 1
        r = r.reshape(1, -1) if single else r
        if r.shape[1] != self.n_nodes:
            raise ValueError("reset must have one entry per vertex")
        out = np.empty_like(r)
        _lib.check(self._lib.hrag_ppr(self._h, r.shape[0], _ptr(r), damping, int(iters), float(tol), _ptr(out)))
        return out[0] if single else out

    def ppr_f64(self, reset, damping: float = 0.5, tol: float = 0.0) -> np.ndarray:
        """``run_ppr`` at PRPACK's accuracy: reset [B, N] (or [N]) -> float64 probabilities, same shape, each column
        within ``tol`` relative L1 error (0 = 1e-10) by a rigorous a-posteriori bound (``hrag_ppr_f64``).  Needs a
        graph loaded from float64 values (``load_graph``, or ``load_graph_csr`` with a float64 ``val``)."""
        r = np.ascontiguousarray(reset, dtype=np.float64)
        single = r.ndim == 1
        r = r.reshape(1, -1) if single else r
        if r.shape[1] != self.n_nodes:
            raise ValueError("reset must have one entry per vertex")
        out = np.empty_like(r)
        _lib.check(self._lib.hrag_ppr_f64(self._h, r.shape[0], _ptr(r), damping, float(tol), _ptr(out)))
        return out[0] if single else out

    def similarity(self, which: int, q) -> np.ndarray:
        """Min-max-normalised scores of every fact (which=0) / passage (which=1): [B, rows] fp32."""
        q = _f32(q)
        rows = self.n_facts if which == 0 else self.n_passages
        out = np.empty((q.shape[0], rows), dtype=np.float32)
        _lib.check(self._lib.hrag_similarity(self._h, which, q.shape[0], _ptr(q), _ptr(out)))
        return out

    def topk_similarity(self, which: int, q, k: int):
        """Top-k raw dot products against the fact (0) / passage (1) embedding matrix: (ids, scores) [B, k]."""
        q = _f32(q)
        ids = np.empty((q.shape[0], k), dtype=np.int32)
        scores = np.empty((q.shape[0], k), dtype=np.float32)
        _lib.check(self._lib.hrag_topk_similarity(self._h, which, q.shape[0], _ptr(q), k, _ptr(ids), _ptr(scores)))
        return ids, scores

    def knn_threshold(self, which: int, q, min_score: float, kmax: int = 128):
        """Rows of embedding matrix ``which`` with dot product >= min_score, best first, at most kmax per query:
        (ids [B, kmax] (-1 padded), scores [B, kmax], n_found [B]); selection fused into the GEMM epilogue."""
        q = _f32(q)
        ids = np.empty((q.shape[0], kmax), dtype=np.int32)
        scores = np.empty((q.shape[0], kmax), dtype=np.float32)
        found = np.empty(q.shape[0], dtype=np.int32)
        _lib.check(self._lib.hrag_knn_threshold(self._h, which, q.shape[0], _ptr(q), float(min_score), kmax, _ptr(ids),
                                                _ptr(scores), _ptr(found)))
        return ids, scores, found

    # ---------------------------------------------------------------- resident self-KNN (synonymy edges)
    def knn_index_update(self, emb, kept_from=None, min_score: float = 0.8, kmax: int = 128) -> int:
        """Keep the self-KNN of ``emb`` ([rows, dim] fp32 unit rows, numpy or a contiguous CUDA tensor on the handle's
        device) on the device (``hrag_knn_index_update``): per row the first ``kmax`` rows with dot product >=
        ``min_score``, best first.  ``kept_from[i]`` (strictly increasing) is the row held before that is now row i,
        for the first ``len(kept_from)`` rows; the rest are new.  ``None`` builds from scratch.  Returns 0 built,
        1 updated, 2 unchanged."""
        if hasattr(emb, "is_cuda"):
            if not (emb.is_cuda and emb.device.index == self.device and emb.is_contiguous()
                    and str(emb.dtype) == "torch.float32" and emb.dim() == 2):
                raise ValueError("device rows must be a contiguous 2-D fp32 CUDA tensor on the handle's device")
            import torch
            torch.cuda.current_stream(self.device).synchronize()
            ptr, (rows, dim), on_dev, keep = C.c_void_p(emb.data_ptr()), tuple(emb.shape), 1, emb
        else:
            keep = _f32(emb)
            if keep.ndim != 2:
                raise ValueError("rows must be a 2-D array")
            ptr, (rows, dim), on_dev = _ptr(keep), keep.shape, 0
        kf = None if kept_from is None else np.ascontiguousarray(kept_from, dtype=np.int64).reshape(-1)
        n_kept = 0 if kf is None else int(kf.shape[0])
        if kf is not None and n_kept == 0:
            kf = np.zeros(1, np.int64)                      # an empty kept_from is not NULL (NULL = build)
        mode = C.c_int32()
        _lib.check(self._lib.hrag_knn_index_update(self._h, int(rows), int(dim), ptr, on_dev, n_kept, _ptr(kf),
                                                   float(min_score), int(kmax), C.byref(mode)))
        del keep                                            # alive until the call has returned
        return int(mode.value)

    def knn_index_info(self) -> Tuple[int, int, int]:
        """(rows, dim, kmax) of the resident self-KNN index, zeros when none is held."""
        rows, dim, kmax = C.c_int64(), C.c_int32(), C.c_int32()
        _lib.check(self._lib.hrag_knn_index_info(self._h, C.byref(rows), C.byref(dim), C.byref(kmax)))
        return int(rows.value), int(dim.value), int(kmax.value)

    def knn_index_read(self):
        """The resident self-KNN lists: (ids [rows, kmax] int32, -1 padded; scores [rows, kmax] fp32, 0 padded)."""
        rows, _, kmax = self.knn_index_info()
        ids = np.empty((rows, kmax), dtype=np.int32)
        scores = np.empty((rows, kmax), dtype=np.float32)
        _lib.check(self._lib.hrag_knn_index_read(self._h, 0, rows, _ptr(ids), _ptr(scores), None))
        return ids, scores

    def knn_index_clear(self):
        """Drop the resident self-KNN index and free its memory."""
        _lib.check(self._lib.hrag_knn_index_clear(self._h))

    def knn_set_memory(self, max_device_bytes: int):
        """The device bytes the self-KNN index's bf16 hi / lo planes (rows x dim x 4 bytes) may take
        (``hrag_knn_set_memory``; 0 = no limit), applied by the next ``knn_index_update``.  Larger planes are kept in
        pinned host memory and streamed through a device ring of at most this many bytes (two slices of a multiple of
        256 rows); the lists stay on the device and are bit for bit those of device planes.  When an update's rows
        cross the budget, or the budget changed, the planes move with one copy."""
        _lib.check(self._lib.hrag_knn_set_memory(self._h, int(max_device_bytes)))

    def knn_planes_info(self) -> dict:
        """Where the self-KNN index's planes are: ``on_host``, the ring's ``slice_rows`` (0 on the device), the planes'
        ``device_bytes`` (the ring when on the host) and the pinned ``host_bytes``."""
        on_host, slice_rows, dev, host = C.c_int(), C.c_int64(), C.c_int64(), C.c_int64()
        _lib.check(self._lib.hrag_knn_planes_info(self._h, C.byref(on_host), C.byref(slice_rows), C.byref(dev),
                                                  C.byref(host)))
        return {"on_host": int(on_host.value), "slice_rows": int(slice_rows.value), "device_bytes": int(dev.value),
                "host_bytes": int(host.value)}

    def bench_sweep(self, batch: int, sweeps: int = 20, method: int = PPR_POWER) -> float:
        ms = C.c_float()
        _lib.check(self._lib.hrag_bench_sweep(self._h, batch, sweeps, method, C.byref(ms)))
        return float(ms.value)

    # ---------------------------------------------------------------- introspection
    @property
    def stream_ptr(self) -> int:
        """cudaStream_t of the handle (wrap with torch.cuda.ExternalStream to record events on it)."""
        return int(self._lib.hrag_stream(self._h) or 0)

    def stats(self) -> dict:
        s = _lib.Stats()
        _lib.check(self._lib.hrag_get_stats(self._h, C.byref(s)))
        return s.as_dict()

    def reset_stats(self):
        _lib.check(self._lib.hrag_reset_stats(self._h))

    def debug_keep_scores(self, keep: bool = True):
        """Make stage A write the raw fact score matrix (tests); the default tensor-core epilogue is fused."""
        _lib.check(self._lib.hrag_debug_keep_scores(self._h, 1 if keep else 0))

    def debug_sim_ctas(self, n: int = 0):
        """Persistent CTAs of the similarity GEMMs (tests, benchmarks): n > 0 for stage_a and the overlapped GEMMs of
        retrieve_resident, n < 0 runs retrieve_resident's chunks without the overlap, 0 restores the defaults."""
        _lib.check(self._lib.hrag_debug_sim_ctas(self._h, int(n)))

    def debug_dense_first_sweep(self, on: bool = True):
        """Make stage B's mixed solves build and sweep the dense first iterate instead of reading the compact right-hand
        side through the slot map (tests, benchmarks: both give the same bytes); False restores the default."""
        _lib.check(self._lib.hrag_debug_dense_first_sweep(self._h, 1 if on else 0))

    def debug_exact_stage_a(self, on: bool = True):
        """Make stage A run the split similarity GEMM over all facts instead of the hi.hi screen and the split rescore
        of its candidates (tests, benchmarks: both give the same bytes); False restores the default."""
        _lib.check(self._lib.hrag_debug_exact_stage_a(self._h, 1 if on else 0))

    def debug_fact_minmax(self) -> np.ndarray:
        """[rows, 2] fp32: the per-query (min, max) fact scores of the last device stage-A chunk (tests)."""
        buf = np.empty((1024, 2), dtype=np.float32)
        n = C.c_int64()
        _lib.check(self._lib.hrag_debug_fact_minmax(self._h, _ptr(buf), buf.shape[0], C.byref(n)))
        return buf[:n.value].copy()

    def debug_scores(self, which: int) -> np.ndarray:
        cols = self.n_facts if which == 0 else self.n_passages
        buf = np.empty(1024 * max(cols, 1), dtype=np.float32)
        n = C.c_int64()
        _lib.check(self._lib.hrag_debug_copy(self._h, which, _ptr(buf), buf.shape[0], C.byref(n)))
        return buf[:n.value].reshape(-1, cols) if cols else buf[:0]

    GRAPH_PLANES = {"row_ptr": (0, np.int32, 1), "cv": (1, np.int32, 2), "val_lo": (2, np.float32, 1),
                    "row_order": (3, np.int32, 1), "long_rows": (4, np.int32, 1), "long_seg_ptr": (5, np.int32, 1),
                    "segs": (6, np.int32, 4)}

    def debug_graph(self, plane: str) -> np.ndarray:
        """A copy of one plane of the loaded graph (``hrag_debug_graph``): cv as [nnz, 2] int32 {col, fp32 bits},
        segs as [n_seg, 4] int32, every other plane 1-D."""
        which, dtype, width = self.GRAPH_PLANES[plane]
        n = C.c_int64()
        _lib.check(self._lib.hrag_debug_graph(self._h, which, None, 0, C.byref(n)))
        buf = np.empty(n.value // np.dtype(dtype).itemsize, dtype=dtype)
        _lib.check(self._lib.hrag_debug_graph(self._h, which, _ptr(buf), n.value, C.byref(n)))
        return buf.reshape(-1, width) if width > 1 else buf

    INDEX_PLANES = {"passage_vid": (0, np.int32), "fact_subj_vid": (1, np.int32), "fact_obj_vid": (2, np.int32),
                    "ent_chunk_count": (3, np.int32), "fact_hi": (4, np.uint16), "fact_lo": (5, np.uint16),
                    "passage_hi": (6, np.uint16), "passage_lo": (7, np.uint16), "fact_f32": (8, np.float32),
                    "passage_f32": (9, np.float32), "edge_src": (10, np.int32), "edge_dst": (11, np.int32),
                    "edge_w": (12, np.float64)}

    def debug_index(self, plane: str, size_only: bool = False):
        """A copy of one plane of the tables, embeddings or resident edge list (``hrag_debug_index``): the embedding
        planes as [rows, dim] (bf16 bits as uint16), every other plane 1-D; ``size_only`` returns its size in bytes."""
        which, dtype = self.INDEX_PLANES[plane]
        n = C.c_int64()
        _lib.check(self._lib.hrag_debug_index(self._h, which, None, 0, C.byref(n)))
        if size_only:
            return n.value
        buf = np.empty(n.value // np.dtype(dtype).itemsize, dtype=dtype)
        _lib.check(self._lib.hrag_debug_index(self._h, which, _ptr(buf), n.value, C.byref(n)))
        return buf.reshape(-1, self.dim) if 4 <= which <= 9 and self.dim else buf


FactFilter = Callable[[int, Sequence[int], Sequence[float]], Sequence[int]]


class B200Retriever:
    """The hot path on raw arrays: graph edge list + tables + embeddings in, top-k passages out.

    ``fact_filter(q, fact_idx, fact_score) -> kept positions`` stands in for the recognition
    memory filter (``rerank.py:108``); ``None`` = identity (what every benchmark uses).
    """

    def __init__(self, n_nodes, edge_src, edge_dst, edge_w, passage_vid, fact_subj_vid, fact_obj_vid,
                 ent_chunk_count, fact_emb, passage_emb, device: int = 0, damping: float = 0.5,
                 linking_top_k: int = 5, passage_node_weight: float = 0.05, retrieval_top_k: int = 200,
                 engine: Optional[Engine] = None):
        self.engine = engine or Engine(device)
        self.engine.load_graph(n_nodes, edge_src, edge_dst, edge_w)
        self.engine.load_tables(passage_vid, fact_subj_vid, fact_obj_vid, ent_chunk_count)
        self.engine.load_embeddings(fact_emb, passage_emb)
        self.damping = damping
        self.linking_top_k = linking_top_k
        self.passage_node_weight = passage_node_weight
        self.retrieval_top_k = retrieval_top_k

    def retrieve(self, q_fact, q_pass, fact_filter: Optional[FactFilter] = None, topk: Optional[int] = None):
        k = self.linking_top_k
        topk = min(topk or self.retrieval_top_k, 2048)
        idx, score, nv = self.engine.stage_a(q_fact, k)
        if fact_filter is not None:
            for q in range(idx.shape[0]):
                keep = list(fact_filter(q, idx[q, :nv[q]].tolist(), score[q, :nv[q]].tolist()))
                kept_i = [idx[q, j] for j in keep]
                kept_s = [score[q, j] for j in keep]
                idx[q] = -1
                idx[q, :len(kept_i)] = kept_i
                score[q, :len(kept_s)] = kept_s
        ids, scores = self.engine.stage_b(q_pass, idx, score, None, self.damping, self.passage_node_weight,
                                          self.linking_top_k, topk)
        return ids, scores, idx, score
