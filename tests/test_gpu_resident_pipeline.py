"""hrag_retrieve_resident over several 1,024-query chunks overlaps chunk c + 1's similarity GEMMs with chunk c's PPR
sweeps on a second stream.  Every kernel still computes what it computes on one stream, so a multi-chunk call must
return bit for bit what the same queries give in single-chunk calls and through stage A + stage B, and count the same
sweeps.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DIM = 64
TOPK = 50
CHUNK = 1024           # queries per chunk of hrag_retrieve_resident at this size (fused stage A, few passages)


@pytest.fixture(scope="module")
def setup():
    import torch
    import hipporag_b200 as hb
    from hipporag_b200 import synth
    kg = synth.make_kg(4000, 40000, seed=11)
    fe = synth.unit_rows(kg.n_facts, DIM, seed=1)
    pe = synth.unit_rows(kg.n_pass, DIM, seed=2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 2600, seed=5)     # a different query in every row of every chunk
    e = hb.Engine(0)
    e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    e.load_embeddings(fe, pe)
    yield e, torch.from_numpy(qf).cuda(), torch.from_numpy(qp).cuda(), qf, qp
    e.close()


def _resident(e, dqf, dqp):
    import torch
    B = dqf.shape[0]
    oi = torch.empty((B, TOPK), dtype=torch.int32, device="cuda")
    os_ = torch.empty((B, TOPK), dtype=torch.float32, device="cuda")
    e.retrieve_resident(dqf, dqp, oi, os_, topk=TOPK)
    torch.cuda.synchronize()
    return oi.cpu().numpy(), os_.cpu().numpy()


def _in_single_chunks(e, dqf, dqp):
    """The same queries in calls of <= CHUNK queries (one chunk each: the sequential path), and their stats."""
    ids, scores, sweeps, columns = [], [], 0, 0
    for q0 in range(0, dqf.shape[0], CHUNK):
        e.reset_stats()
        i, s = _resident(e, dqf[q0:q0 + CHUNK], dqp[q0:q0 + CHUNK])
        st = e.stats()
        ids.append(i)
        scores.append(s)
        sweeps += st["ppr_sweeps"]
        columns += st["ppr_columns"]
    return np.concatenate(ids), np.concatenate(scores), sweeps, columns


def _assert_same(got, want, what):
    assert np.array_equal(got[0], want[0]), f"{what}: ids differ"
    assert np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32)), f"{what}: scores differ"


@pytest.mark.parametrize("B", [2600, 1025])      # three chunks with a ragged last one; a last chunk of one query
def test_multi_chunk_call_equals_single_chunk_calls(setup, B):
    e, dqf, dqp, _, _ = setup
    want_ids, want_scores, want_sweeps, want_columns = _in_single_chunks(e, dqf[:B], dqp[:B])
    for rep in range(3):
        e.reset_stats()
        got = _resident(e, dqf[:B], dqp[:B])
        st = e.stats()
        _assert_same(got, (want_ids, want_scores), f"B = {B}, call {rep}")
        assert st["ppr_sweeps"] == want_sweeps and st["ppr_columns"] == want_columns, (rep, st)
    # the debug read-back of the passage scores shows the last chunk's rows
    last = e.debug_scores(1)
    q_last = (B - 1) // CHUNK * CHUNK
    _resident(e, dqf[q_last:B], dqp[q_last:B])
    assert last.shape[0] == B - q_last
    assert np.array_equal(last.view(np.uint32), e.debug_scores(1).view(np.uint32))


def test_multi_chunk_call_equals_stage_a_plus_stage_b(setup):
    e, dqf, dqp, qf, qp = setup
    got = _resident(e, dqf, dqp)
    idx, score, _ = e.stage_a(qf, 5)
    want = e.stage_b(qp, idx, score, None, topk=TOPK)     # identity recognition-memory filter
    _assert_same(got, want, "stage A + stage B")
