/* hrag_b200.h -- C ABI of libhrag_b200.so: HippoRAG's online retrieval hot path on H100 (sm_90a).
 *
 * The reference (OSU-NLP-Group/HippoRAG) is pure Python and has no FFI of its own; the
 * boundary this library replaces is a set of methods on the `HippoRAG` object.  Each entry
 * point below names the reference code it stands in for (paths under
 * the reference's src/hipporag/).  INTEGRATION.md shows the ctypes binding a maintainer
 * would add on the reference side.
 *
 * Conventions: every function returns 0 on success, non-zero on failure
 * (hrag_last_error() gives the message).  Host buffers are caller-owned and C-contiguous;
 * device memory is handle-owned.  One handle drives ONE GPU (one process per GPU); a handle
 * is not thread-safe, distinct handles are independent.  There is no CPU fallback: with no
 * CUDA device hrag_create() fails.
 */
#ifndef HRAG_B200_H
#define HRAG_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct hrag_handle hrag_t;

/* PPR solver variants (both sweep the same CSR SpMM kernel). */
#define HRAG_PPR_POWER     0  /* z <- a P z + v            (Neumann / power iteration)        */
#define HRAG_PPR_CHEBYSHEV 1  /* Chebyshev semi-iteration on the same fixed point (default)   */

/* PPR state precision. */
#define HRAG_PPR_FP32   0     /* fp32 state, batch width ppr_batch                                   */
#define HRAG_PPR_MIXED  1     /* fp16 state (width 32) + one fp32 iterative-refinement step: same   */
                              /* accuracy as fp32, ~half the gathered bytes per query; batches of   */
                              /* <= 16 columns, and dampings whose single refinement round cannot   */
                              /* reach `tol`, run the fp32 solver                                   */

/* Similarity precision modes. */
#define HRAG_SIM_FP32     0   /* SIMT fp32 FMA kernel (exact fp32 products)                  */
#define HRAG_SIM_BF16X3   1   /* wgmma bf16 hi/lo split, all 4 products, fp32-faithful (default)   */
#define HRAG_SIM_BF16     2   /* wgmma single bf16 pass (fast mode, NOT the parity mode)      */

typedef struct hrag_stats {
    double ms_sim_fact;      /* stage A: query x fact similarity (K2)                 */
    double ms_select_fact;   /* stage A: min/max + top-k facts                         */
    double ms_sim_passage;   /* stage B: query x passage similarity (K2)               */
    double ms_seed;          /* stage B: seed / reset-vector build (K3)                */
    double ms_ppr;           /* stage B: all PPR sweeps (K1)                           */
    double ms_topk;          /* stage B: passage gather + top-k (K4)                   */
    double ms_comm;          /* sharded mode: exchange time                            */
    int64_t ppr_sweeps;      /* sweeps executed since the last reset                   */
    int64_t ppr_columns;     /* sum over sweeps of the batch width B                   */
    int64_t kernel_launches; /* kernels of this library launched since the last reset  */
    int64_t h2d_bytes;
    int64_t d2h_bytes;
    double ppr_residual;     /* last mixed-solver call: measured relative L1 residual of the fp16 first solve; */
                             /* last hrag_ppr_f64 call: max over its columns of ||r||_1 / ||v||_1 after the    */
                             /* final refinement round (r = v - (I - damping P) x, fp64)                       */
    double ppr_error_bound;  /* a-posteriori bound on the relative L1 error of the PPR vectors of that call:   */
                             /* mixed solver: ppr_residual x the predicted contraction of the refinement round; */
                             /* hrag_ppr_f64: 2 ppr_residual / (1 - damping), rigorous (no model constant)     */
    int64_t stage_a_fallbacks; /* stage-A chunks whose hi.hi screen could not prove its candidates and that    */
                               /* reran the split GEMM over all facts (read at the end of each stage call)    */
} hrag_stats_t;

const char* hrag_last_error(void);
const char* hrag_version(void);

/* Binds a handle to device_ids[0].  n_devices must be 1: multi-GPU runs use one process
 * (and one handle) per GPU, joined by hrag_comm_init().  shard_mode: 0 = replicas
 * (every rank holds the whole graph), 1 = node-range sharding. */
int hrag_create(const int* device_ids, int n_devices, int shard_mode, hrag_t** out);
void hrag_destroy(hrag_t* h);

/* Node-range sharding (SURVEY.md 8(e)): fills a 128-byte NCCL unique id (rank 0), then
 * every rank joins.  The id travels through the host's own process group. */
int hrag_comm_unique_id(void* id128);
int hrag_comm_init(hrag_t* h, const void* id128, int rank, int world);

/* Optional, before the graph load: rank r owns rows [bounds[r], bounds[r + 1]) (bounds[0] = 0, bounds[world] = N) instead
 * of equal row counts -- a partition balanced by work (non-zeros + 4 per row) keeps the ranks in step when some row
 * ranges are much denser than others (the passage rows).  The COO loaders derive it by themselves (every rank sees the
 * whole edge list); a caller of hrag_load_graph_csr passes it explicitly. */
int hrag_comm_set_row_bounds(hrag_t* h, const int64_t* bounds, int world);

/* Fused sweep + exchange for node-range sharding (after hrag_comm_init and the graph load): every
 * rank exports one 64-byte CUDA IPC handle of its PPR state, the host gathers the `world` handles
 * (rank order) and every rank imports them.  From then on the mixed-precision sweep stores its output
 * rows straight into the peers' buffers over NVLink and publishes an epoch flag -- no all-gather. */
int hrag_p2p_export(hrag_t* h, void* handle64);
int hrag_p2p_import(hrag_t* h, const void* handles, int world);

/* The graph HippoRAG.run_ppr walks (HippoRAG.py:1709-1749) as the CSR of P = W D^-1:
 * row i lists (j, W[i,j]/s_j) of the summed symmetric weights of the igraph multigraph that
 * add_new_edges builds (HippoRAG.py:1189-1223).  With node-range sharding a rank passes the
 * rows [row_lo, row_hi) it owns (row_ptr has row_hi-row_lo+1 entries, columns stay global);
 * replicas pass row_lo = 0, row_hi = n_nodes. */
int hrag_load_graph_csr(hrag_t* h, int64_t n_nodes, int64_t row_lo, int64_t row_hi, int64_t nnz,
                        const int64_t* row_ptr, const int32_t* col, const float* val);

/* Same as hrag_load_graph_csr from float64 values of P (the graph of HippoRAG.py:1189-1223 as run_ppr's
 * PRPACK call sees it, :1736-1743): the fp32 plane every solver sweeps is fp32(val), bitwise what
 * hrag_load_graph_csr stores for those values, and a second plane lo = fp32(val - fp32(val)) keeps P to
 * ~2^-48 relative for hrag_ppr_f64 (4 more bytes per non-zero of HBM).  hrag_load_graph_coo keeps the lo
 * plane as well; a graph loaded through hrag_load_graph_csr has none. */
int hrag_load_graph_csr_f64(hrag_t* h, int64_t n_nodes, int64_t row_lo, int64_t row_hi, int64_t nnz,
                            const int64_t* row_ptr, const int32_t* col, const double* val);

/* Same graph from the igraph-style undirected multigraph edge list itself
 * (graph.get_edgelist() + graph.es["weight"]): every edge (src, dst, w) contributes w to W[src,dst]
 * and W[dst,src]; parallel edges sum (add_fact_edges emits (s,o) and (o,s), HippoRAG.py:907-910);
 * edges with w <= 0 carry nothing; columns are divided by the vertex strength.  The endpoints are
 * checked on the host; the library then uploads the list and builds the CSR on the GPU (no scipy
 * needed by a C caller), byte for byte what a sequential build gives: parallel edges summed in input
 * order, strengths summed in column order, fp64 division.  The graph keeps the fp64 lo plane of
 * hrag_load_graph_csr_f64.  With node-range sharding every rank passes the full edge list and keeps
 * its own row range.  Scratch while it runs: about 100 bytes of device memory per edge. */
int hrag_load_graph_coo(hrag_t* h, int64_t n_nodes, int64_t n_edges, const int32_t* src, const int32_t* dst,
                        const double* w);

/* Same as hrag_load_graph_coo from an edge list already in this handle's GPU memory (device pointers,
 * n_edges entries each, ready to read: the caller has synchronised the stream that wrote them).  The
 * endpoints are checked on the device; a rejected list leaves the handle as it was.  Nothing is kept
 * from the arrays once the call returns. */
int hrag_load_graph_coo_device(hrag_t* h, int64_t n_nodes, int64_t n_edges, const int32_t* d_src,
                               const int32_t* d_dst, const double* d_w);

/* Integer tables equivalent to the dicts prepare_retrieval_objects builds
 * (HippoRAG.py:1287-1389): passage_vid[p] = passage_node_idxs[p] (:1333);
 * fact_subj_vid / fact_obj_vid = node_name_to_vertex_idx["entity-"+md5(phrase)] of each
 * fact's subject / object, -1 when absent (:1591-1597); ent_chunk_count[v] =
 * len(ent_node_to_chunk_ids[key]) (:1598-1601, 0 when absent). */
int hrag_load_tables(hrag_t* h, int64_t n_passages, const int32_t* passage_vid, int64_t n_facts,
                     const int32_t* fact_subj_vid, const int32_t* fact_obj_vid,
                     const int32_t* ent_chunk_count);

/* fact_embeddings (which = 0, HippoRAG.py:1345) / passage_embeddings (which = 1, :1343):
 * [rows, dim] fp32, C order.  on_device != 0: emb is a device pointer. */
int hrag_load_embeddings(hrag_t* h, int which, int64_t rows, int32_t dim, const float* emb,
                         int on_device);

/* Streamed upload for a matrix too large to keep in fp32 next to its bf16 hi/lo planes (BASELINE config #5:
 * 27.5 M facts x 1024 = 113 GB of fp32): _begin allocates only the planes of the tensor-core similarity
 * (rows x dim x 4 bytes); every _chunk converts fp32 rows [row0, row0 + n_rows) (host or device pointer) and
 * forgets them.  HRAG_SIM_FP32 is then unavailable for that matrix.  With node-range sharding a rank keeps
 * only the rows of its own fact slice and ignores the rest of a chunk. */
int hrag_load_embeddings_begin(hrag_t* h, int which, int64_t rows, int32_t dim);
int hrag_load_embeddings_chunk(hrag_t* h, int which, int64_t row0, int64_t n_rows, const float* emb,
                               int on_device);

/* Device memory of the fact planes (the bf16 hi / lo planes of fact_embeddings, HippoRAG.py:1345, that stage A's
 * similarity reads, rows x dim x 4 bytes), set before the fact embeddings are loaded and applied by every later fact
 * load.  0 (the default) or a budget of at least the planes keeps them resident.  A smaller budget keeps them in
 * library-owned pinned host memory, byte for byte the planes a resident load builds, and streams them through a
 * device ring of at most max_device_bytes: two slices, each a multiple of 256 rows (a budget below two 256-row slices,
 * 2 x 256 x dim x 4 bytes, fails the load).  Every entry then returns bit for bit what the resident planes give:
 * hrag_stage_a streams the planes once per call (per 256 MB of bf16 query splits: 65,536 queries at dim 1024), as does
 * the stage A of hrag_retrieve_resident, which runs for the whole call before its chunks (the get_fact_scores /
 * rerank_facts of HippoRAG.py:459-470 for all queries); hrag_similarity / hrag_topk_similarity (which = 0) stream
 * them once per query chunk.  With host planes: no fp32 fact rows are kept (HRAG_SIM_FP32 is unavailable for the
 * facts, as after a streamed upload); hrag_load_embeddings rejects fact rows on the device; hrag_knn_threshold
 * (which = 0), the update entries and sharded handles (world > 1) are rejected; h2d_bytes counts the streamed plane
 * bytes.  A reload or hrag_destroy frees the pinned memory.  The passage planes are always resident. */
int hrag_set_fact_memory(hrag_t* h, int64_t max_device_bytes);
/* The budget covers the fact planes only.  Resident planes of at least 65,536 facts also take the stage-A screen's
 * scratch at the first stage-A call (one GPU, HRAG_SIM_BF16X3): about 0.6 GB at 2.75 M facts x 768 for a
 * 1,024-query chunk (per m-tile staging planes 48 x 256 x d x 4 bytes, per query and 256-fact tile 16 bytes, per
 * m-tile and fact 4 bytes). */
/* What the last fact load chose: on_host (1 = pinned host planes, 2 = hi plane resident and lo plane in pinned host
 * memory, see hrag_set_fact_placement), the ring's slice_rows (0 when resident), the device bytes of the fact planes
 * (the ring, the resident planes, or the hi plane plus the lo ring) and the pinned host bytes (0 when resident). */
int hrag_fact_planes_info(hrag_t* h, int* on_host, int64_t* slice_rows, int64_t* device_bytes, int64_t* host_bytes);

/* Where a fact load puts the planes when they exceed the hrag_set_fact_memory budget; set before the fact embeddings
 * are loaded and applied by every later fact load.  HRAG_FACT_PLANES_BY_BUDGET (the default) is the rule above.
 * HRAG_FACT_LO_ON_HOST keeps the hi plane resident and only the lo plane in library-owned pinned host memory (mapped,
 * so kernels read it over PCIe):
 *   - planes within the budget, or budget 0: resident, as by default;
 *   - else, when the hi plane (rows x dim x 2 bytes) plus a lo ring of two 256-row slices (2 x 256 x dim x 2 bytes)
 *     fit the budget: hi resident, lo on the host, and a ring of two lo slices, each the largest multiple of 256 rows
 *     that fits the rest of the budget (hrag_fact_planes_info: on_host = 2);
 *   - else the load fails, naming the hi plane's bytes and the budget (nothing falls back to both planes on the host).
 * Stage A then runs the stage-A screen (one GPU, HRAG_SIM_BF16X3, >= 65,536 facts, linking_top_k <= 8): the hi.hi
 * screen reads the resident hi plane, and only the lo rows of the staged candidates cross PCIe (counted in
 * h2d_bytes).  A query chunk whose screen cannot prove its candidates reruns the split product with the lo plane
 * streamed through the ring (stage_a_fallbacks counts it).  Every other route that needs every lo row (fewer than
 * 65,536 facts, linking_top_k > 8, hrag_debug_keep_scores, hrag_debug_exact_stage_a, hrag_similarity /
 * hrag_topk_similarity with which = 0) streams the lo plane only; HRAG_SIM_BF16 reads nothing from the host.  The
 * outputs are byte for byte those of resident planes.  Rejected as with host planes: fact rows on the device for
 * hrag_load_embeddings, HRAG_SIM_FP32 for the facts, hrag_knn_threshold (which = 0), the update entries,
 * hrag_index_export, and sharded handles (world > 1).  The budget does not cover the screen's scratch (staging planes,
 * per m-tile and fact 4 bytes) nor its per-chunk partials, 88 bytes per query and 256-fact tile, which grow with the
 * fact count: under this placement the screen's query chunk is the largest multiple of 128 (at most 1,024) whose
 * partials stay within 1 GB, 1,024 queries at 2.75 M facts, 128 at 17 M. */
#define HRAG_FACT_PLANES_BY_BUDGET 0
#define HRAG_FACT_LO_ON_HOST       1
int hrag_set_fact_placement(hrag_t* h, int placement);

/* Incremental updates of a loaded index: what HippoRAG.index() (HippoRAG.py:262-335: the stores append, igraph
 * add_vertices / add_edges, :1187, :1220) and HippoRAG.delete() (:337-411: the stores pop in place, igraph
 * delete_vertices compacts in order, :408) do to the arrays this handle mirrors, applied on the device without a
 * reload.  After any sequence of updates the handle holds, byte for byte, what a fresh load (hrag_load_graph_coo,
 * hrag_load_tables, hrag_load_embeddings) of the resulting arrays gives: the graph planes are rebuilt from the
 * resident edge list by the loaders' own builder, tables and embedding planes are appended to or compacted in order.
 * Every input is checked before the handle is touched (a rejected call leaves it as it was); a call that fails after
 * that (out of memory) leaves no graph, tables or embeddings rather than a half-updated index.
 *
 * on != 0 before a COO graph load: the handle keeps the edge list as given (int32 src, int32 dst, fp64 w: 16 bytes
 * of HBM per edge, edges with w <= 0 or NaN included), which the update entries need.  The update entries reject
 * handles without it (not mutable, graph loaded from a CSR), node-range-sharded handles (world > 1) and embedding
 * matrices whose fp32 rows are borrowed from the caller (hrag_load_embeddings with on_device != 0). */
int hrag_set_mutable(hrag_t* h, int on);

/* Optional: sizes the capacity of the edge list (edges), ent_chunk_count (nodes), the fact tables and fact embedding
 * planes (facts) and the passage table and planes (passages) up front, so that no later append copies a plane into
 * a larger allocation (which holds both copies for a moment).  Without it capacity grows by half at a time. */
int hrag_index_reserve(hrag_t* h, int64_t nodes, int64_t edges, int64_t facts, int64_t passages);

/* HippoRAG.index(): appends n_new_nodes vertices (ids N .. N + n_new_nodes - 1), n_new_edges edges (endpoints in
 * the grown range), n_new_passages rows of passage_vid, n_new_facts rows of fact_subj_vid / fact_obj_vid (-1 =
 * absent) -- as hrag_load_tables takes them -- with their embedding rows fact_emb [n_new_facts, dim] and
 * passage_emb [n_new_passages, dim]; ent_chunk_count is the whole new table [N + n_new_nodes].  dim must be the
 * index's.  Only the new rows are uploaded and split into the bf16 planes.  Host arrays, except where on_device sets
 * HRAG_DEVICE_EDGES (src / dst / w are device pointers, checked on the device), HRAG_DEVICE_FACT_EMB or
 * HRAG_DEVICE_PASSAGE_EMB (the embedding rows are device pointers; they are copied, not borrowed). */
#define HRAG_DEVICE_EDGES        1
#define HRAG_DEVICE_FACT_EMB     2
#define HRAG_DEVICE_PASSAGE_EMB  4
int hrag_index_append(hrag_t* h, int64_t n_new_nodes, int64_t n_new_edges, const int32_t* src, const int32_t* dst,
                      const double* w, int64_t n_new_passages, const int32_t* passage_vid, int64_t n_new_facts,
                      const int32_t* fact_subj_vid, const int32_t* fact_obj_vid, const int32_t* ent_chunk_count,
                      int32_t dim, const float* fact_emb, const float* passage_emb, int on_device);

/* HippoRAG.delete(): removes the vertices del_nodes (sorted, unique) and the fact rows del_facts (sorted, unique),
 * host arrays.  The remaining vertices are renumbered in order, edges with a deleted endpoint go and the others keep
 * their order (parallel edges are summed in input order), passage rows whose vertex went are dropped and the others
 * relabelled, fact subjects / objects are relabelled (a deleted vertex becomes -1), and the embedding rows follow
 * their passages and facts, compacted in place.  ent_chunk_count is the whole new table [N - n_del_nodes]. */
int hrag_index_delete(hrag_t* h, int64_t n_del_nodes, const int32_t* del_nodes, int64_t n_del_facts,
                      const int32_t* del_facts, const int32_t* ent_chunk_count);

/* One loaded index served to several processes on the same GPU through CUDA IPC (a rag_qa service runs one
 * worker process per HippoRAG object; each would otherwise load and hold its own copy of the index).
 *
 * hrag_index_export (the owner: a handle with graph, tables and embeddings loaded) writes a self-describing blob of
 * *size bytes; blob == NULL only reports *size, cap is the room at blob.  The blob begins with an 8-byte magic and a
 * uint32 layout version, and carries the owner's device UUID and pid, the index's sizes, and one CUDA IPC handle per
 * allocation that query code only reads: the graph planes (row_ptr, cv, row_order, the long-row segment tables,
 * val_lo), the four seed tables, and the bf16 planes and owned fp32 rows of both embedding matrices; plus an 8-byte
 * attach counter.  Rejected: no index loaded, fact planes in pinned host memory (hrag_set_fact_memory; that memory
 * is this process's), world > 1, fp32 rows borrowed from the caller (device load), an attached handle.  Exporting
 * again returns the same allocations.  While exported the owner serves every call as before, but its loads (graph,
 * tables, embeddings, streamed embeddings) and hrag_index_append / _delete / _reserve are rejected, leaving the
 * handle and its results unchanged.  hrag_index_unexport is rejected while a handle is attached; after it the
 * handle is an ordinary one again (blobs exported before it no longer attach).  To update a shared index: have the
 * workers detach, unexport, update, export again.
 *
 * The owner process must outlive every attached handle: freeing an allocation another process maps is undefined
 * in CUDA, so hrag_destroy of an owner with live attachments frees everything except the exported allocations, which
 * the process exit releases.
 *
 * hrag_index_attach maps the blob's allocations into a fresh handle (no index loaded, world == 1) in another process
 * on the same physical GPU, without a copy.  Rejected: a blob of another version or size (truncated), another GPU
 * (UUID), a handle that already holds an index, and a blob exported by the calling process (cudaIpcOpenMemHandle
 * cannot open a handle its own process exported).  The attached handle serves every call an owner serves
 * (stages A / B, hrag_stage_b_f64, hrag_ppr, hrag_ppr_f64, hrag_similarity, hrag_topk_similarity,
 * hrag_knn_threshold, hrag_retrieve_resident, the debug reads, its own synonymy KNN index) with the same results;
 * its streams, solver state, scratch, captured solves and stats are its own.  Loads and updates are rejected until
 * hrag_index_detach, which closes the mappings and leaves an ordinary empty handle; hrag_destroy detaches too.
 * Attached handles time-slice the GPU with the owner; they do not run concurrently.
 *
 * hrag_index_share_info: role (0 none, 1 owner, 2 attached), the live attach count (0 for role 0), imported_bytes
 * = the bytes of the shared allocations (exported by an owner, mapped by an attached handle; 0 for role 0) and
 * owned_bytes = the device bytes this handle allocated itself (an owner's include its shared allocations). */
int hrag_index_export(hrag_t* h, void* blob, int64_t cap, int64_t* size);
int hrag_index_unexport(hrag_t* h);
int hrag_index_attach(hrag_t* h, const void* blob, int64_t size);
int hrag_index_detach(hrag_t* h);
int hrag_index_share_info(hrag_t* h, int* role, int64_t* n_attached, int64_t* imported_bytes, int64_t* owned_bytes);

/* Engine knobs that are not BaseConfig fields (SURVEY.md 5).  ppr_iters > 0 pins the sweep count of the
 * fp32 solver; by default it is derived from the damping factor (see hrag_stage_b). */
int hrag_set_options(hrag_t* h, int ppr_method, int ppr_iters, int ppr_batch, int sim_mode);
/* precision: HRAG_PPR_FP32 / HRAG_PPR_MIXED (-1 keeps); sweeps1 / sweeps2 > 0 pin the fp16 Chebyshev sweeps
 * before / after the residual step of the mixed solver (default: derived from damping, 8 / 7 at 0.5). */
int hrag_set_ppr_precision(hrag_t* h, int precision, int sweeps1, int sweeps2);

/* Stage A = get_fact_scores + the argsort of rerank_facts (HippoRAG.py:1427-1465,
 * 1683-1688) for B queries: top_idx[b, :] = the k best fact rows (best first; tie -> lower
 * row), top_score = their min-max-normalised scores (misc_utils.py:130-139), n_valid[b] =
 * min(k, n_facts).  k = linking_top_k (config_utils.py:184) in [1, 32]: k <= 8 is selected in the GEMM
 * epilogue, larger k by an exact radix select on the materialised scores.  Host buffers. */
int hrag_stage_a(hrag_t* h, int32_t B, const float* q_fact, int32_t k, int32_t* top_idx,
                 float* top_score, int32_t* n_valid);

/* Stage B = dense_passage_retrieval + graph_search_with_fact_entities + run_ppr + the slice
 * in _build_retrieval_result (HippoRAG.py:1467-1502, 1544-1656, 1709-1749, 501-507) for B
 * queries.  kept_fact_idx[b, :] are the fact rows that survived the recognition-memory
 * filter (-1 padded), kept_fact_score their normalised scores; a query with no kept fact or
 * dpr_only[b] != 0 takes the DPR fallback (:467-469).  out_ids index passage_node_keys
 * order (:1745), out_scores are PPR probabilities (or min-maxed DPR scores on fallback),
 * sorted by (score desc, id asc).  k_facts <= 32.  Host buffers.
 *
 * iters, tol: PRPACK iterates to 1e-10 whatever the damping (HippoRAG.py:1736-1743; damping is
 * config_utils.py:192).  Here tol = requested relative L1 accuracy of each PPR vector (0 = 1e-6, the level
 * the fp32 outputs can show) and the sweep counts are DERIVED from it: the iteration operator has its
 * spectrum in [-damping, damping], so Chebyshev contracts by damping / (1 + sqrt(1 - damping^2)) per sweep
 * (14 fp32 sweeps, or 8 + 1 + 7 fp16 sweeps with refinement, at damping 0.5; 32 fp32 sweeps at 0.85).
 * iters > 0 pins the count instead.  The mixed solver measures the residual of its first solve and the call
 * FAILS (status 4) when residual x predicted contraction misses 10 x tol. */
int hrag_stage_b(hrag_t* h, int32_t B, const float* q_pass, const int32_t* kept_fact_idx,
                 const float* kept_fact_score, int32_t k_facts, const uint8_t* dpr_only,
                 float damping, float passage_node_weight, int32_t link_top_k, int32_t topk,
                 int32_t iters, float tol, int32_t* out_ids, float* out_scores);

/* hrag_stage_b at PRPACK's accuracy: what the reference's retrieve() computes (graph_search_with_fact_entities ->
 * run_ppr, HippoRAG.py:1544-1656, 1709-1749), float64 to 1e-10.  The reset vector is built on the device in the
 * reference's dtypes (phrase weights fp32(score) / fp32(chunk count), averaged in float64; passage weights
 * fp32(minmax(dpr)) x fp32(passage_node_weight); summed in float64), solved as hrag_ppr_f64 solves (per sub-batch of
 * <= 16 queries), and the passage scores are gathered and ranked in float64: out_scores [B, topk] float64, sorted by
 * (score desc, id asc) exactly, -1 / 0 padded when topk > passages.  DPR-fallback rows are stage B's fp32 min-maxed
 * scores, widened.  Arguments as in hrag_stage_b, except: damping is float64; tol is the relative L1 error bound of
 * every PPR vector (0 = 1e-10, below 1e-13 is rejected); status 4 when 4 refinement rounds do not reach tol (the
 * outputs are then unspecified); ppr_residual / ppr_error_bound of hrag_get_stats report the call.  Needs a graph
 * loaded through hrag_load_graph_csr_f64 or hrag_load_graph_coo; fails on a node-range-sharded handle (world > 1). */
int hrag_stage_b_f64(hrag_t* h, int32_t B, const float* q_pass, const int32_t* kept_fact_idx,
                     const float* kept_fact_score, int32_t k_facts, const uint8_t* dpr_only, double damping,
                     float passage_node_weight, int32_t link_top_k, int32_t topk, double tol, int32_t* out_ids,
                     double* out_scores);

/* The rule hrag_stage_b / hrag_ppr apply to (damping, tol, iters) for a batch of `batch` columns with the default engine
 * options, as a pure host function (no device needed): which solver runs (use_mixed: fp16 state + refinement, batches > 16
 * whose single refinement round reaches tol), the fp32 solver's sweep count, the mixed solver's two counts, and the
 * predicted relative L1 error of the result. */
int hrag_plan_sweeps(float damping, float tol, int32_t iters, int32_t batch, int32_t* use_mixed, int32_t* fp32_sweeps,
                     int32_t* mixed_sweeps1, int32_t* mixed_sweeps2, double* predicted_error);

/* Whole retrieve() loop body for B queries with the identity recognition-memory filter,
 * inputs and outputs resident in HBM (device pointers): the device-timed benchmark leg.  Runs in chunks of up to
 * 1,024 queries; on one GPU the similarity GEMMs of chunk c + 1 run on a second stream while chunk c's PPR sweeps
 * run, with the same results as one chunk per call. */
int hrag_retrieve_resident(hrag_t* h, int32_t B, const float* d_q_fact, const float* d_q_pass,
                           float damping, float passage_node_weight, int32_t link_top_k,
                           int32_t topk, int32_t iters, float tol, int32_t* d_out_ids, float* d_out_scores);

/* run_ppr's numeric core (HippoRAG.py:1735-1743) for B reset vectors: reset is [B, N]
 * (host), NaN/negative entries count as 0; out is [B, N] probabilities.  iters / tol as in hrag_stage_b. */
int hrag_ppr(hrag_t* h, int32_t B, const float* reset, float damping, int32_t iters, float tol, float* out);

/* run_ppr at PRPACK's accuracy (HippoRAG.py:1735-1743: float64 reset, float64 scores, tolerance 1e-10) for B
 * reset vectors: reset is [B, N] float64 (host), NaN/negative entries count as 0; out is [B, N] float64
 * probabilities; damping is taken in float64 as PRPACK takes it.  Iterative refinement: fp32 sweeps solve each correction, the residual is recomputed in fp64
 * against the fp64 operator, until the rigorous bound 2 ||r||_1 / ((1 - damping) ||v||_1) on the relative L1
 * error of every column is <= tol (0 = 1e-10; below 1e-13 is rejected).  Status 4 when 4 rounds do not reach
 * tol.  ppr_residual / ppr_error_bound of hrag_get_stats report the call.  Needs a graph loaded through
 * hrag_load_graph_csr_f64 or hrag_load_graph_coo; fails on a node-range-sharded handle (world > 1). */
int hrag_ppr_f64(hrag_t* h, int32_t B, const double* reset, double damping, double tol, double* out);

/* Full score vectors for code that calls get_fact_scores (which = 0, HippoRAG.py:1427-1465)
 * or dense_passage_retrieval (which = 1, :1467-1502) directly: out[b, :] = min-max-normalised
 * <q[b], E[:, :]>, [B, rows] on the host. */
int hrag_similarity(hrag_t* h, int which, int32_t B, const float* q, float* out);

/* Top-k raw similarities (SURVEY.md 8(f)-2: the index-time synonymy KNN, utils/embed_utils.py:6-94
 * = blocked torch.mm + torch.topk): for each of B queries the k (<= 2048) rows of the fact
 * (which = 0) / passage (which = 1) embedding matrix with the largest dot product, sorted
 * (score desc, row asc); out_ids / out_scores are [B, k] (host), -1 / 0 padded when k > rows. */
int hrag_topk_similarity(hrag_t* h, int which, int32_t B, const float* q, int32_t k, int32_t* out_ids,
                         float* out_scores);

/* The KNN as add_synonymy_edges actually consumes it (HippoRAG.py:1003-1018: walk the neighbours in score order,
 * stop at the first score < synonymy_edge_sim_threshold or after 100 accepted ones): for each of B queries the rows
 * of embedding matrix `which` with dot product >= min_score, best first (score desc, row asc), at most kmax (<= 512) of
 * them; the rest of out_ids / out_scores [B, kmax] is -1 / 0.  The threshold is applied inside the GEMM epilogue -- the
 * [B, rows] score matrix is never written.  n_found[b] = how many rows cleared the threshold; n_found[b] > 512 means
 * the list of that query overflowed and it must be re-run through hrag_topk_similarity. */
int hrag_knn_threshold(hrag_t* h, int which, int32_t B, const float* q, float min_score, int32_t kmax,
                       int32_t* out_ids, float* out_scores, int32_t* n_found);

/* The self-KNN of add_synonymy_edges (HippoRAG.py:980-992: every entity against every entity) kept on the device
 * between calls and updated in place when the entity store changes.  The handle holds one such index, independent of
 * the retrieval index (no graph or mutable handle needed; hrag_index_append / hrag_index_delete leave it alone): the
 * bf16 hi / lo planes of its rows and, per row, the first kmax rows with dot product >= min_score, best first (score
 * desc, row asc) -- after every call exactly what hrag_knn_threshold(rows, rows, min_score, kmax) on a fresh handle,
 * with the rows whose n_found exceeds 512 redone through hrag_topk_similarity and cut at min_score, gives for the rows
 * of this call, bit for bit (split bf16 x 4 products whatever hrag_set_options chose).
 *
 * emb: [rows, dim] fp32 rows in the NEW order (host, or a device pointer if on_device), dim % 8 == 0.  Row i < n_kept
 * is the row held at kept_from[i] (strictly increasing), rows >= n_kept are new: only the new keys are scored against
 * the kept rows, and only new rows and lists that lost a listed key without holding every key >= min_score are scored
 * against all keys.  Kept rows are verified against the planes held: a changed vector rebuilds.  kept_from == NULL, no
 * index held, or a changed min_score, kmax (in [1, 512]) or dim builds from scratch.  *mode: 0 built, 1 updated, 2
 * unchanged (no GEMM ran).  Every argument is checked before the index is touched (a rejected call leaves it as it
 * was); a failure after that (out of memory) clears it.  Rejected on a node-range-sharded handle (world > 1).  Device
 * memory: 4 dim + 8 pad4(kmax + 1) bytes per row, capacity grown by half at a time (the planes' share bounded by
 * hrag_knn_set_memory). */
int hrag_knn_index_update(hrag_t* h, int64_t rows, int32_t dim, const float* emb, int on_device, int64_t n_kept,
                          const int64_t* kept_from, float min_score, int32_t kmax, int32_t* mode);
/* Device memory of the index's bf16 hi / lo planes (rows x dim x 4 bytes), applied by every later
 * hrag_knn_index_update.  0 (the default) or a budget of at least the planes keeps them on the device as above.  A
 * smaller budget keeps them in library-owned pinned host memory and streams them through a device ring of two halves,
 * each a multiple of 256 rows, within the budget; an update then stages its query rows on the device in passes of up
 * to 65,536 rows and streams the keys once per pass.  The lists (8 pad4(kmax + 1) bytes per row) stay on the device and
 * every list is bit for bit what resident planes give.  Placement follows the rows of each update: when they cross the
 * budget, in either direction, or the budget changed, the planes move with one copy and the lists are kept.  An update
 * whose planes would need a ring below two 256-row slices (2 x 256 x dim x 4 bytes) is rejected, leaving the index as
 * it was.  There is no automatic mode: free device memory on a shared GPU would pick another placement from run to
 * run.  A non-zero budget is rejected on a node-range-sharded handle (world > 1). */
int hrag_knn_set_memory(hrag_t* h, int64_t max_device_bytes);
/* Where the index's planes are: on_host (1 = pinned host planes), the ring's slice_rows (0 when on the device), the
 * device bytes of the planes (the ring, or the planes' capacity) and the pinned host bytes (capacity; 0 on the
 * device). */
int hrag_knn_planes_info(hrag_t* h, int* on_host, int64_t* slice_rows, int64_t* device_bytes, int64_t* host_bytes);
/* Rows [row0, row0 + n) of the index: ids / scores [n, kmax] (host, -1 / 0 padded), n_valid[n] (may be NULL). */
int hrag_knn_index_read(hrag_t* h, int64_t row0, int64_t n, int32_t* ids, float* scores, int32_t* n_valid);
/* What the index holds: *rows, *dim and *kmax (all 0 when no index is held). */
int hrag_knn_index_info(hrag_t* h, int64_t* rows, int32_t* dim, int32_t* kmax);
/* Drops the index and frees its memory. */
int hrag_knn_index_clear(hrag_t* h);

/* K1 micro-benchmark: runs `sweeps` SpMM sweeps at batch width B on resident synthetic
 * state and returns the average milliseconds per sweep (CUDA events on the launch stream).
 * method: 0 power / 1 Chebyshev (fp32 state), 2 fp16 state with a dense rhs, 3 fp16 state with the
 * compact rhs of stage B (needs hrag_load_tables), 4 the paired sweep of two such sub-batches ([N, 2, 32] state, time
 * per paired sweep); 5 / 6 the paired FIRST sweep of a stage-B solve (plain, no prev), 5 gathering the dense first
 * iterate, 6 the compact rhs through the slot maps of the passages. */
int hrag_bench_sweep(hrag_t* h, int32_t B, int32_t sweeps, int32_t method, float* ms_per_sweep);

/* The CUDA stream (cudaStream_t) every call of this handle is ordered on: a call starts after the work already on
 * it, and the work it runs on the handle's other streams is joined back into it before the call returns, so a
 * caller can bracket calls with its own CUDA events. */
void* hrag_stream(hrag_t* h);

/* Stage times are summed CUDA-event spans per stream.  hrag_retrieve_resident overlaps the similarity stages of
 * one chunk of queries with the PPR of the previous chunk, so there the stage times can add up to more than the
 * call's elapsed time. */
int hrag_get_stats(hrag_t* h, hrag_stats_t* out);
int hrag_reset_stats(hrag_t* h);
/* Raw device buffers for tests/benchmarks: which = 0 fact scores of the last stage A
 * sub-batch, 1 passage scores of the last stage B sub-batch. */
int hrag_debug_copy(hrag_t* h, int which, float* host_out, int64_t max_elems, int64_t* n_written);
/* The per-query (min, max) fact scores of the last device stage-A chunk (<= 1024 rows of 2 floats; 0 rows after a
 * stage A over host fact planes). */
int hrag_debug_fact_minmax(hrag_t* h, float* host_out, int64_t max_rows, int64_t* n_rows);
/* One plane of the loaded graph, byte for byte (tests compare the ingest planes): plane = 0 row_ptr int32[n_rows + 1],
 * 1 cv int2[nnz], 2 val_lo fp32[nnz] (empty without the fp64 operator), 3 row_order int32[n_rows], 4 long_rows
 * int32[n_long], 5 long_seg_ptr int32[n_long + 1] (empty when n_long = 0), 6 segs int4[n_seg].  *n_written = the
 * plane's size in bytes; host_out = NULL only reports it. */
int hrag_debug_graph(hrag_t* h, int plane, void* host_out, int64_t max_bytes, int64_t* n_written);
/* One plane of the loaded tables, embeddings or edge list, byte for byte (tests compare updated and fresh handles):
 * plane = 0 passage_vid int32[P], 1 fact_subj_vid int32[F], 2 fact_obj_vid int32[F], 3 ent_chunk_count int32[N],
 * 4 / 5 the bf16 hi / lo planes of the fact embeddings [F, dim], 6 / 7 those of the passage embeddings [P, dim],
 * 8 / 9 the fp32 fact / passage rows [rows, dim] (empty when not held), 10 edge src int32[E], 11 edge dst int32[E],
 * 12 edge weight fp64[E] (the list a mutable handle keeps).  *n_written = the plane's size in bytes; host_out =
 * NULL only reports it. */
int hrag_debug_index(hrag_t* h, int plane, void* host_out, int64_t max_bytes, int64_t* n_written);
/* keep != 0: stage A materialises the fact score matrix even in the tensor-core modes (whose
 * default epilogue selects min/max/top-k in registers and never writes scores). */
int hrag_debug_keep_scores(hrag_t* h, int keep);
/* Persistent CTAs of the similarity GEMMs (tests and benchmarks; the results do not depend on it).  n > 0: hrag_stage_a
 * runs its GEMMs on n CTAs, and a multi-chunk hrag_retrieve_resident runs the overlapped GEMMs of chunk c + 1 on n
 * CTAs instead of the count derived from the shapes; n < 0: hrag_retrieve_resident runs its chunks one after the
 * other without the overlap; n = 0 restores the defaults. */
int hrag_debug_sim_ctas(hrag_t* h, int n);
/* on != 0: stage B's mixed solves scatter their right-hand side into a dense first iterate and sweep it, as
 * node-range-sharded handles do, instead of reading it through the slot map (tests and benchmarks compare the two
 * forms; the results are the same bit for bit); 0 restores the default. */
int hrag_debug_dense_first_sweep(hrag_t* h, int on);
/* on != 0: stage A runs the split GEMM over all facts instead of the hi.hi screen and the split rescore of its
 * candidates (tests and benchmarks compare the two; the results are the same bit for bit); 0 restores the default. */
int hrag_debug_exact_stage_a(hrag_t* h, int on);

#ifdef __cplusplus
}
#endif
#endif /* HRAG_B200_H */
