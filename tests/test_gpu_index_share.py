"""One index shared between processes on one GPU (hrag_index_export / hrag_index_attach): a handle in another process
attached to an owner's index must return, byte for byte, what the owner returns; the owner and the attached handles
must reject what would change or free the shared memory; the attach count, the memory accounting and the drop-in's
attach= path must hold.

Children are spawned processes serving commands over a Pipe (``_child``); every child is joined in a ``finally``
with a timeout, then terminated and joined, so none outlives its test.  Owners are closed only after their children
have exited (a child's exit detaches it).
"""
import contextlib
import multiprocessing as mp

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TIMEOUT = 300
SIM_BF16X3, SIM_BF16 = 1, 2


# ------------------------------------------------------------------------------ the child process
def _call(eng, call):
    """Run one (method, args, kwargs) on an Engine; results as a tuple of numpy arrays (None for setters)."""
    name, args, kw = call
    if name == "retrieve_resident":
        import torch
        qf, qp = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in args)
        B, topk = qf.shape[0], kw["topk"]
        ids = torch.empty((B, topk), dtype=torch.int32, device="cuda")
        scores = torch.empty((B, topk), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        eng.retrieve_resident(qf, qp, ids, scores, **kw)
        return ids.cpu().numpy(), scores.cpu().numpy()
    out = getattr(eng, name)(*args, **kw)
    if out is None:
        return None
    return tuple(np.array(o) for o in out) if isinstance(out, tuple) else (np.array(out),)


def _dropin(kg_fields, fact_emb, passage_emb, q_fact, q_pass, queries, blob):
    from tests import fake_hipporag
    fake_hipporag.install_stub_package()
    import hipporag_b200
    from hipporag_b200 import synth
    rag = fake_hipporag.FakeRag(synth.SynthKG(**kg_fields), fact_emb, passage_emb, q_fact, q_pass, queries)
    hipporag_b200.accelerate(rag, device=0, cache=False, attach=blob)
    sols = rag.retrieve(queries, num_to_retrieve=50)
    info = rag._b200_state["engine"].share_info()
    try:
        rag.index(["another document"])
        index_error = None
    except hipporag_b200.HragError as e:
        index_error = str(e)
    return [(s.docs, np.asarray(s.doc_scores)) for s in sols], info, index_error


def _child(conn):
    """Command loop: ("engine",) makes the child's Engine; ("run", calls) / ("repeat", call, n) run calls;
    ("dropin", ...) runs the drop-in; any other command is an Engine method.  Replies ("ok", out) or ("err", msg)."""
    import hipporag_b200 as hb
    eng = None
    try:
        while True:
            cmd, *args = conn.recv()
            if cmd == "exit":
                break
            try:
                if cmd == "engine":
                    eng, out = hb.Engine(0), None
                elif cmd == "run":
                    out = [_call(eng, c) for c in args[0]]
                elif cmd == "repeat":
                    out = [_call(eng, args[0]) for _ in range(args[1])]
                elif cmd == "dropin":
                    out = _dropin(*args)
                else:
                    out = getattr(eng, cmd)(*args)
                conn.send(("ok", out))
            except Exception as e:   # reported to the parent, which decides
                conn.send(("err", f"{type(e).__name__}: {e}"))
    finally:
        if eng is not None:
            eng.close()          # an attached handle detaches
        conn.close()


class Child:
    def __init__(self):
        ctx = mp.get_context("spawn")
        self.conn, theirs = ctx.Pipe()
        self.proc = ctx.Process(target=_child, args=(theirs,), daemon=True)
        self.proc.start()
        theirs.close()

    def ask(self, cmd, *args):
        self.conn.send((cmd, *args))
        assert self.conn.poll(TIMEOUT), f"child: no answer to {cmd} within {TIMEOUT} s"
        return self.conn.recv()

    def ok(self, cmd, *args):
        status, out = self.ask(cmd, *args)
        assert status == "ok", f"{cmd}: {out}"
        return out

    def err(self, cmd, *args):
        status, out = self.ask(cmd, *args)
        assert status == "err", f"{cmd} was accepted"
        return out

    def stop(self):
        try:
            self.conn.send(("exit",))
        except (OSError, ValueError):
            pass
        self.proc.join(TIMEOUT)
        if self.proc.is_alive():
            self.proc.terminate()
            self.proc.join(30)
        self.conn.close()


@contextlib.contextmanager
def children(n):
    kids = []
    try:
        for _ in range(n):
            kids.append(Child())
        for c in kids:
            c.ok("engine")
        yield kids
    finally:
        for c in kids:
            c.stop()


# ------------------------------------------------------------------------------ owners
def _load(eng, kg, fe, pe):
    eng.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    eng.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    eng.load_embeddings(fe, pe)
    return eng


def _inputs(kg, pe, qf, qp, seed):
    rng = np.random.default_rng(seed)
    B = 40
    kept_idx = rng.integers(0, kg.n_facts, size=(B, 5)).astype(np.int32)
    kept_idx[3, 2:] = -1
    kept_idx[7] = -1                                       # no kept fact: DPR fallback
    kept_score = rng.random((B, 5)).astype(np.float32)
    dpr = np.zeros(B, np.uint8)
    dpr[[1, 20, 33]] = 1                                   # DPR-only rows
    reset = np.zeros((20, kg.n_nodes), np.float64)
    for b in range(20):
        reset[b, rng.integers(0, kg.n_nodes, size=6)] = rng.random(6)
    # knn_threshold: about 100 hits over 8 queries, none near the 512 a list keeps (beyond that a list holds
    # whichever hits arrived first)
    thr = float(np.sort((qp[:8] @ pe.T).ravel())[-100])
    return dict(qf=qf, qp=qp, ki=kept_idx, ks=kept_score, dpr=dpr, reset=reset, thr=thr)


def _calls(d):
    calls = []
    for mode in (SIM_BF16X3, SIM_BF16):
        calls.append(("set_options", (), {"sim_mode": mode}))
        calls += [("stage_a", (d["qf"][:40], k), {}) for k in (5, 8, 9, 32)]
    calls.append(("set_options", (), {"sim_mode": SIM_BF16X3}))
    for B in (12, 40):                                     # fp32 solver (B <= 16), paired mixed solves (B > 16)
        calls.append(("stage_b", (d["qp"][:B], d["ki"][:B], d["ks"][:B], d["dpr"][:B]), {"topk": 50}))
    calls.append(("stage_b_f64", (d["qp"][:12], d["ki"][:12], d["ks"][:12], d["dpr"][:12]), {"topk": 50}))
    calls.append(("ppr", (d["reset"].astype(np.float32),), {}))
    calls.append(("ppr_f64", (d["reset"],), {}))
    calls += [("similarity", (w, q[:8]), {}) for w, q in ((0, d["qf"]), (1, d["qp"]))]
    calls += [("topk_similarity", (w, q[:8], 20), {}) for w, q in ((0, d["qf"]), (1, d["qp"]))]
    calls.append(("knn_threshold", (1, d["qp"][:8], d["thr"]), {"kmax": 64}))
    calls.append(("retrieve_resident", (d["qf"], d["qp"]), {"topk": 50}))   # > 1,024 queries: two chunks
    return calls


def _same(got, want, what):
    if want is None:
        assert got is None, what
        return
    assert len(got) == len(want), what
    for i, (a, b) in enumerate(zip(got, want)):
        a, b = np.asarray(a), np.asarray(b)
        assert a.shape == b.shape and a.dtype == b.dtype, f"{what}[{i}]: {a.shape} {a.dtype} != {b.shape} {b.dtype}"
        assert a.tobytes() == b.tobytes(), f"{what}[{i}]: {int((a != b).sum())} entries differ"


@pytest.fixture(scope="module")
def synthetic():
    """A power-law graph whose hubs are long rows (the per-handle segment partials are exercised)."""
    import hipporag_b200 as hb
    from hipporag_b200 import synth
    kg = synth.make_kg(20000, 200000, seed=3, topology="powerlaw")
    fe, pe = synth.unit_rows(kg.n_facts, 64, seed=1), synth.unit_rows(kg.n_pass, 64, seed=2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 1300, seed=4)
    owner = _load(hb.Engine(0), kg, fe, pe)
    assert owner.debug_graph("long_rows").size > 0
    yield dict(kg=kg, fe=fe, pe=pe, owner=owner, d=_inputs(kg, pe, qf, qp, 5))
    owner.close()


@pytest.fixture(scope="module")
def musique(golden):
    import hipporag_b200 as hb
    from hipporag_b200 import synth
    g = golden
    n, P = int(g["n_nodes"]), int(g["passage_vid"].shape[0])
    kg = synth.SynthKG(n_nodes=n, n_ent=n - P, n_pass=P, edge_src=g["edge_src"], edge_dst=g["edge_dst"],
                       edge_w=g["edge_w"], passage_vid=g["passage_vid"], fact_subj_vid=g["fact_subj_vid"],
                       fact_obj_vid=g["fact_obj_vid"], ent_chunk_count=g["ent_chunk_count"],
                       fact_passage=np.zeros(g["fact_subj_vid"].shape[0], np.int32))
    qf = np.resize(g["q_fact"], (1100, g["q_fact"].shape[1])).astype(np.float32)     # two retrieve_resident chunks
    qp = np.resize(g["q_pass"], (1100, g["q_pass"].shape[1])).astype(np.float32)
    owner = _load(hb.Engine(0), kg, g["fact_emb"], g["passage_emb"])
    yield dict(kg=kg, fe=g["fact_emb"], pe=g["passage_emb"], owner=owner, d=_inputs(kg, g["passage_emb"], qf, qp, 6), g=g)
    owner.close()


# ------------------------------------------------------------------------------ outputs and memory
@pytest.mark.parametrize("which", ["synthetic", "musique"])
def test_attached_outputs_equal_owner(request, which):
    w = request.getfixturevalue(which)
    owner = w["owner"]
    blob = owner.export_index()
    calls = _calls(w["d"])
    with children(1) as (child,):
        assert child.ok("share_info") == {"role": "none", "n_attached": 0, "imported_bytes": 0, "owned_bytes": 0}
        child.ok("attach", blob)
        mine, theirs = owner.share_info(), child.ok("share_info")
        assert mine["role"] == "owner" and mine["n_attached"] == 1
        assert theirs["role"] == "attached" and theirs["n_attached"] == 1
        assert theirs["imported_bytes"] == mine["imported_bytes"] > 0
        n_seg = owner.debug_graph("segs").shape[0]
        assert theirs["owned_bytes"] == n_seg * 64 * 4          # its own segment partials, nothing of the index
        got = child.ok("run", calls)
        child.ok("detach")
        assert owner.share_info()["n_attached"] == 0
    want = [_call(owner, c) for c in calls]
    n_found = want[[c[0] for c in calls].index("knn_threshold")][2]
    assert 0 < n_found.sum() and n_found.max() <= 512
    for c, a, b in zip(calls, got, want):
        _same(a, b, f"{which} {c[0]}")
    owner.unexport()
    assert owner.share_info()["role"] == "none"


def test_two_children_attached_at_once(synthetic):
    owner, d = synthetic["owner"], synthetic["d"]
    call = ("stage_b", (d["qp"][:40], d["ki"][:40], d["ks"][:40], d["dpr"][:40]), {"topk": 50})
    blob = owner.export_index()
    with children(2) as kids:
        for c in kids:
            c.ok("attach", blob)
        assert owner.share_info()["n_attached"] == 2
        for c in kids:                                      # both loops in flight at once
            c.conn.send(("repeat", call, 10))
        outs = []
        for c in kids:
            assert c.conn.poll(TIMEOUT)
            status, out = c.conn.recv()
            assert status == "ok", out
            outs.append(out)
    assert owner.share_info()["n_attached"] == 0
    want = _call(owner, call)
    for out in outs:
        for got in out:
            _same(got, want, "concurrent stage_b")
    owner.unexport()


# ------------------------------------------------------------------------------ lifetime rules
def test_owner_rules(synthetic):
    import hipporag_b200 as hb
    kg, fe, pe, d = synthetic["kg"], synthetic["fe"], synthetic["pe"], synthetic["d"]
    owner = _load(hb.Engine(0, mutable=True), kg, fe, pe)
    call = ("stage_b", (d["qp"][:40], d["ki"][:40], d["ks"][:40], d["dpr"][:40]), {"topk": 50})
    before = _call(owner, call)
    blob = owner.export_index()
    cc = np.append(kg.ent_chunk_count, 0).astype(np.int32)
    rejected = {
        "load_graph": lambda: owner.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w),
        "load_graph_csr": lambda: owner.load_graph_csr(kg.n_nodes, *hb.build_transition_csr(
            kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)),
        "load_tables": lambda: owner.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid,
                                                 kg.ent_chunk_count),
        "load_embeddings": lambda: owner.load_embeddings(fe, pe),
        "load_embeddings_streamed": lambda: owner.load_embeddings_streamed(1, pe.shape[0], 64, [(0, pe)]),
        "append": lambda: owner.append(1, ent_chunk_count=cc),
        "delete": lambda: owner.delete(facts=[0], ent_chunk_count=kg.ent_chunk_count),
        "reserve": lambda: owner.reserve(facts=kg.n_facts + 10),
    }
    try:
        with children(1) as (child,):
            child.ok("attach", blob)
            assert owner.share_info()["n_attached"] == 1
            with pytest.raises(hb.HragError, match="still attached"):
                owner.unexport()
            with pytest.raises(hb.HragError, match="still attached"):
                owner.close()
            for name, fn in rejected.items():
                with pytest.raises(hb.HragError, match="exported"):
                    fn()
            _same(_call(owner, call), before, "owner stage_b while exported")
            _same(child.ok("run", [call])[0], before, "attached stage_b")
            child.ok("detach")
        assert owner.share_info()["n_attached"] == 0
        owner.unexport()
        assert owner.share_info()["role"] == "none"
        owner.append(1, ent_chunk_count=cc)
        assert owner.n_nodes == kg.n_nodes + 1
    finally:
        owner.close()


def test_attached_handle_rules(synthetic):
    owner, kg, fe, pe = synthetic["owner"], synthetic["kg"], synthetic["fe"], synthetic["pe"]
    d = synthetic["d"]
    blob = owner.export_index()
    call = ("stage_a", (d["qf"][:40], 5), {})
    with children(1) as (child,):
        child.ok("attach", blob)
        for cmd, args in (("load_graph", (kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)),
                          ("load_tables", (kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)),
                          ("load_embeddings", (fe, pe)),
                          ("reserve", (0, 0, kg.n_facts + 10, 0)),
                          ("append", (1, (), (), (), (), (), (), np.append(kg.ent_chunk_count, 0))),
                          ("delete", ((), (), kg.ent_chunk_count))):
            assert "attached" in child.err(cmd, *args), cmd
        assert "attached" in child.err("export_index")
        child.ok("detach")
        assert child.ok("share_info")["role"] == "none"
        child.ok("load_graph", kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
        child.ok("load_tables", kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
        child.ok("load_embeddings", fe, pe)
        got = child.ok("run", [call])[0]
    _same(got, _call(owner, call), "stage_a after detach and a load")
    owner.unexport()


# ------------------------------------------------------------------------------ rejections
def test_export_rejections(synthetic):
    import hipporag_b200 as hb
    kg, fe, pe = synthetic["kg"], synthetic["fe"], synthetic["pe"]
    empty = hb.Engine(0)
    try:
        with pytest.raises(hb.HragError, match="no index loaded"):
            empty.export_index()
    finally:
        empty.close()
    host = _load(hb.Engine(0, fact_device_bytes=2 * 256 * 64 * 4 + 100), kg, fe, pe)
    try:
        assert host.fact_planes_info()["on_host"] == 1
        with pytest.raises(hb.HragError, match="pinned host memory"):
            host.export_index()
        assert host.share_info()["role"] == "none"
    finally:
        host.close()


def test_attach_rejections(synthetic):
    import hipporag_b200 as hb
    owner, kg = synthetic["owner"], synthetic["kg"]
    blob = owner.export_index()
    wrong_version = blob[:8] + (int.from_bytes(blob[8:12], "little") + 1).to_bytes(4, "little") + blob[12:]
    same = hb.Engine(0)
    try:
        with pytest.raises(hb.HragError, match="exported by this process"):
            same.attach(blob)
        assert same.share_info()["role"] == "none"
    finally:
        same.close()
    with children(1) as (child,):
        assert "truncated" in child.err("attach", blob[:-8])
        assert "version" in child.err("attach", wrong_version)
        assert "not a blob" in child.err("attach", b"\0" * len(blob))
        child.ok("load_graph", kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
        assert "already holds an index" in child.err("attach", blob)
        assert child.ok("share_info")["role"] == "none"
    assert owner.share_info()["n_attached"] == 0
    owner.unexport()


# ------------------------------------------------------------------------------ the drop-in
def test_dropin_attach_equals_owner(musique):
    from tests import fake_hipporag
    fake_hipporag.install_stub_package()
    import hipporag_b200
    from hipporag_b200 import synth
    g, kg = musique["g"], musique["kg"]
    queries = [f"question {i}" for i in range(g["q_fact"].shape[0])]
    args = (g["fact_emb"], g["passage_emb"], g["q_fact"], g["q_pass"], queries)
    rag = fake_hipporag.FakeRag(kg, *args)
    hipporag_b200.accelerate(rag, device=0, cache=False)
    want = rag.retrieve(queries, num_to_retrieve=50)
    blob = hipporag_b200.share(rag)
    eng = rag._b200_state["engine"]
    fields = {k: getattr(kg, k) for k in synth.SynthKG.__dataclass_fields__}
    try:
        with children(1) as (child,):
            got, info, index_error = child.ok("dropin", fields, *args, blob)
            assert info["role"] == "attached"
            assert eng.share_info()["n_attached"] == 1
        assert index_error and "attached" in index_error
        assert eng.share_info()["n_attached"] == 0
        for (docs, scores), w in zip(got, want):
            assert docs == w.docs
            _same((scores,), (np.asarray(w.doc_scores),), "doc_scores")
        # another index: the fingerprint differs and nothing is attached
        other = dict(fields, edge_w=np.asarray(kg.edge_w) * 2.0)
        rag2 = fake_hipporag.FakeRag(synth.SynthKG(**other), *args)
        hipporag_b200.accelerate(rag2, device=0, cache=False, attach=blob)
        with pytest.raises(hipporag_b200.HragError, match="fingerprint"):
            rag2.retrieve(queries[:2], num_to_retrieve=10)
        with pytest.raises(ValueError):
            hipporag_b200.accelerate(rag2, device=0, cache=False, attach=blob, incremental=True)
    finally:
        eng.unexport()
        eng.close()
