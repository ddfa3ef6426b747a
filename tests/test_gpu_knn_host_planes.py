"""The synonymy KNN index with its planes in pinned host memory (hrag_knn_set_memory): after every update of a sequence
its lists (ids, scores, n_valid) must equal, bit for bit, those of a handle whose planes are on the device, and at the
end what a fresh handle's threshold KNN plus knn.py's overflow redo gives over the final rows.

Rows are +-1/8 in d = 64, so every score is an exact multiple of 1/64 and no score lies near the threshold 0.8 (51/64 <
0.8 < 52/64): the GEMM's float32 cut and the redo's float64 cut agree.  Planted clusters share 58 coordinates with a
template (score >= 52/64 among themselves): cluster A has more than 512 members, cluster B more than 128, spread over
every slice, so the candidate buffers and the overflow redo cross slice edges.  Exact copies of one row sit on both
sides of slice edges, so equal scores (1.0) meet there.  A ring slice is a multiple of 256 rows: the budgets below give
3, 4 and 33 slices over the 8,300 rows of the build.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DIM = 64
THR = 0.8
ROWS = 8300
ROW_BYTES = DIM * 4                  # hi + lo planes of one row


def budget(slice_rows):
    """The device bytes of a ring of two slice_rows-row halves."""
    return 2 * slice_rows * ROW_BYTES


BUDGETS = {3: budget(2816), 4: budget(2304), 33: budget(256)}       # slices over ROWS rows
DUP_AT = (255, 256, 2303, 2304, 2815, 2816, 5119, 5120, 5631, 5632, 8191, 8192)


@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


class Data:
    """Rows drawn from one generator: random rows, members of clusters A / B and copies of one duplicate row."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.templates = self.rng.choice([-1.0, 1.0], size=(3, DIM))

    def rows(self, n, a=0, b=0, dups=()):
        """n rows: a of cluster A and b of cluster B at random rows other than `dups`, copies of the duplicate row
        at `dups`."""
        x = self.rng.choice([-1.0, 1.0], size=(n, DIM))
        pos = self.rng.permutation(np.setdiff1d(np.arange(n), dups))
        x[pos[:a], :58] = self.templates[0, :58]
        x[pos[a:a + b], :58] = self.templates[1, :58]
        x[list(dups)] = self.templates[2]
        return (x / 8).astype(np.float32)

    def initial(self):
        return self.rows(ROWS, a=600, b=200, dups=DUP_AT)


class Store:
    """Rows changed the way EmbeddingStore changes them: appends, in-order deletes."""

    def __init__(self, rows):
        self.rows = rows

    def change(self, delete=(), append=None):
        keep = np.ones(self.rows.shape[0], bool)
        keep[list(delete)] = False
        kept_from = np.flatnonzero(keep)
        self.rows = self.rows[keep]
        if append is not None:
            self.rows = np.concatenate([self.rows, append])
        return kept_from


def read(eng):
    """(ids, scores, n_valid) of the whole index through hrag_knn_index_read."""
    from hipporag_b200 import _lib
    rows, _, kmax = eng.knn_index_info()
    ids = np.empty((rows, kmax), np.int32)
    sc = np.empty((rows, kmax), np.float32)
    nv = np.empty(rows, np.int32)
    p = lambda a: C.c_void_p(a.ctypes.data)
    _lib.check(eng._lib.hrag_knn_index_read(eng._h, 0, rows, p(ids), p(sc), p(nv)))
    return ids, sc, nv


def assert_same(got, want, what):
    ids, sc, nv = got
    wids, wsc, wnv = want
    assert ids.shape == wids.shape, what
    bad = np.nonzero((ids != wids).any(axis=1) | (sc.view(np.uint32) != wsc.view(np.uint32)).any(axis=1)
                     | (nv != wnv))[0]
    assert bad.size == 0, f"{what}: {bad.size} rows differ, first {bad[:5]}"


def per_call(hb, keys, kmax):
    """A fresh handle's threshold KNN + overflow redo over `keys` (knn.py's recipe): (ids, scores, n_valid)."""
    M = keys.shape[0]
    e = hb.Engine(0)
    try:
        e.load_embeddings(keys, keys[:1])
        ids, sc, found = e.knn_threshold(0, keys, THR, kmax)
        redo = np.nonzero(found > 512)[0]
        if redo.size:
            rid, rsc = e.topk_similarity(0, keys[redo], int(min(kmax, M)))
            for j, q in enumerate(redo):
                keep = rsc[j] >= np.float32(THR)
                ids[q], sc[q] = -1, 0.0
                ids[q, :keep.sum()] = rid[j][keep]
                sc[q, :keep.sum()] = rsc[j][keep]
        return ids, sc, (ids >= 0).sum(axis=1).astype(np.int32)
    finally:
        e.close()


class Pair:
    """A handle with host planes (budget) and one with device planes, updated alike."""

    def __init__(self, hb, budget_bytes, kmax):
        self.host, self.dev, self.kmax, self.budget = hb.Engine(0), hb.Engine(0), kmax, budget_bytes
        self.host.knn_set_memory(budget_bytes)

    def update(self, rows, kept_from=None, what=""):
        mode = self.host.knn_index_update(rows, kept_from, THR, self.kmax)
        want = self.dev.knn_index_update(rows, kept_from, THR, self.kmax)
        assert mode == want, what
        assert_same(read(self.host), read(self.dev), what)
        return mode

    def close(self):
        self.host.close()
        self.dev.close()


def _sequence(hb, pair, data):
    store = Store(data.initial())
    assert pair.update(store.rows, what="build") == 0
    info = pair.host.knn_planes_info()
    assert info["on_host"] == 1 and info["device_bytes"] <= pair.budget
    assert pair.dev.knn_planes_info()["on_host"] == 0
    # 300 new rows over the slice edge at 8,448, 100 of them joining cluster A and 50 cluster B
    kf = store.change(append=data.rows(300, a=100, b=50))
    assert pair.update(store.rows, kf, "append") == 1
    ca = np.flatnonzero((store.rows[:, :58] == data.templates[0, :58] / 8).all(axis=1))
    cb = np.flatnonzero((store.rows[:, :58] == data.templates[1, :58] / 8).all(axis=1))
    assert ca.size > 600 and cb.size > 200
    deletes = (("delete at the front", lambda n: list(range(10)) + [int(ca[0])]),
               ("delete in the middle", lambda n: list(range(4000, 4100)) + [int(i) for i in ca[ca > 4100][:20]]
                + [int(i) for i in cb[cb > 4100][:5]]),
               ("delete at the tail", lambda n: list(range(n - 25, n))))
    for what, gone in deletes:
        kf = store.change(delete=sorted(set(gone(store.rows.shape[0]))))
        assert pair.update(store.rows, kf, what) == 1
    n = store.rows.shape[0]
    gone = sorted(set(data.rng.choice(n, 50, replace=False).tolist()))
    kf = store.change(delete=gone, append=data.rows(200, a=80, b=10))
    assert pair.update(store.rows, kf, "delete + append") == 1
    kf = store.change()
    assert pair.update(store.rows, kf, "unchanged") == 2
    changed = store.rows.copy()
    changed[100, 60] = -changed[100, 60]
    store.rows = changed
    assert pair.update(store.rows, np.arange(store.rows.shape[0]), "changed kept vector") == 0
    assert_same(read(pair.host), per_call(hb, store.rows, pair.kmax), "fresh threshold KNN + redo")


@pytest.mark.parametrize("kmax", [1, 100, 128, 512])
@pytest.mark.parametrize("n_slices", [3, 4, 33])
def test_host_planes_equal_device_planes(hb, n_slices, kmax):
    pair = Pair(hb, BUDGETS[n_slices], kmax)
    try:
        _sequence(hb, pair, Data(seed=n_slices * 1000 + kmax))
        assert -(-ROWS // pair.host.knn_planes_info()["slice_rows"]) == n_slices
    finally:
        pair.close()


def test_migration_both_ways(hb):
    data = Data(seed=7)
    pair = Pair(hb, 1000 * ROW_BYTES, 128)      # planes of 1,000 rows; slices of 256 rows when over it
    try:
        store = Store(data.rows(900, a=300, b=150))
        pair.update(store.rows, what="build under the budget")
        assert pair.host.knn_planes_info() == {"on_host": 0, "slice_rows": 0, "device_bytes": 2 * 900 * DIM * 2,
                                               "host_bytes": 0}
        kf = store.change(append=data.rows(200, a=40))
        pair.update(store.rows, kf, "append over the budget")
        info = pair.host.knn_planes_info()
        assert info["on_host"] == 1 and info["slice_rows"] == 256 and info["device_bytes"] == budget(256)
        assert info["host_bytes"] >= 1100 * ROW_BYTES
        kf = store.change(delete=list(range(0, 600, 2)))
        pair.update(store.rows, kf, "delete under the budget")
        assert pair.host.knn_planes_info()["on_host"] == 0
        # a budget changed while the index is held applies at the next update, also an unchanged one
        pair.host.knn_set_memory(budget(256))
        assert pair.update(store.rows, store.change(), "budget lowered") == 2
        assert pair.host.knn_planes_info()["on_host"] == 1
        kf = store.change(delete=[3, 400], append=data.rows(30, a=10))
        pair.update(store.rows, kf, "update on host planes")
        pair.host.knn_set_memory(0)
        assert pair.update(store.rows, store.change(), "budget lifted") == 2
        assert pair.host.knn_planes_info()["on_host"] == 0
        kf = store.change(delete=[0], append=data.rows(5))
        pair.update(store.rows, kf, "update after moving back")
    finally:
        pair.close()


def test_rejections_leave_the_index(hb):
    from hipporag_b200 import HragError
    data = Data(seed=11)
    eng = hb.Engine(0)
    try:
        with pytest.raises(HragError, match="budget must be >= 0"):
            eng.knn_set_memory(-1)
        eng.knn_set_memory(budget(256))
        rows = data.rows(1500, a=600)
        assert eng.knn_index_update(rows, None, THR, 128) == 0
        before, info = read(eng), eng.knn_planes_info()
        assert info["on_host"] == 1
        eng.knn_set_memory(budget(256) - 1)            # below two 256-row slices
        more = np.concatenate([rows, data.rows(10)])
        with pytest.raises(HragError, match="hrag_knn_set_memory budget of .* is below the"):
            eng.knn_index_update(more, np.arange(1500), THR, 128)
        with pytest.raises(HragError, match="below the"):
            eng.knn_index_update(more, None, THR, 128)
        assert eng.knn_planes_info() == info and eng.knn_index_info() == (1500, DIM, 128)
        assert_same(read(eng), before, "after the rejected updates")
        eng.knn_set_memory(budget(256))
        with pytest.raises(HragError, match="kept_from"):
            eng.knn_index_update(more, np.arange(1, 1502), THR, 128)
        assert_same(read(eng), before, "after a rejected kept_from")
        assert eng.knn_index_update(more, np.arange(1500), THR, 128) == 1
        assert_same(read(eng), per_call(hb, more, 128), "after the next update")
    finally:
        eng.close()


def test_accelerate_drop_in_with_a_budget():
    from tests import fake_hipporag
    from tests.test_accelerate_knn_incremental import EntityRag, _entities, _run
    fake_hipporag.install_stub_package()
    import hipporag_b200
    rng = np.random.default_rng(5)
    a, b, c = _entities(rng, 1500, 0), _entities(rng, 400, 1500), _entities(rng, 300, 1900)
    ops = [("index", a), ("index", b), ("delete", [f"entity {i}" for i in (0, 7, 800, 1501, 1899)]), ("index", c)]
    results = []
    for knn_bytes in (None, budget(256)):
        rag = EntityRag()
        hipporag_b200.accelerate(rag, device=0, incremental=True, cache=False, knn_device_bytes=knn_bytes)
        ran, edges = [], []
        for op, spec in ops:
            _run(rag, [(op, spec)])
            ran.append(rag._b200_state.get("last_knn"))
            edges.append(dict(rag.node_to_node_stats))
        rag.add_synonymy_edges()
        ran.append(rag._b200_state["last_knn"])
        eng = rag._b200_state["engine"]
        assert eng.knn_planes_info()["on_host"] == (knn_bytes is not None)
        results.append((ran, edges))
        eng.close()
    assert results[0][0] == results[1][0] == ["built", "updated", "updated", "updated", "unchanged"]
    assert results[0][1] == results[1][1] and len(results[0][1][-1]) > 1000
