"""Exact (score, start) ties: the reference keeps its top-K in a heapq of (score, stack) tuples
(traceweaver_v3.py:305-307) and sorts it with list.sort(reverse=True) (:461).  Two different spans
with the same start_mus compare neither-smaller (spans.py:51), so which of two equal entries
survives and where it lands is decided by heapq's sift order.  The oracle replays heapq; the
engine's sequential paths (tw_core.cuh topk_offer / topk_finish, stepped here on the CPU) must
give the same lists, and so must its lane-parallel path, which hands an in-span with a tie among its
six best back to the sequential replay.  Inputs: millisecond clocks (alibaba-shaped and DAGs of up to
eight callees), parallel eps, heavy overlap."""
from functools import partial

import numpy as np
import pytest

import skip_synth
from oracle import tw_oracle
from emul_backend import EmulBatch
from traceweaver_b200 import synth
from traceweaver_b200.batch import build_batch, build_batch_from_blocks

CASES = {
    "par3_ms": ("ali_par3", 3, 160, 100.0, 1000),
    "chain2_ms": ("ali_chain2", 3, 200, 100.0, 1000),
    "leaf_ms": ("ali_leaf", 3, 200, 100.0, 1000),
    "leaf_dense_ms": ("ali_leaf", 4, 300, 300.0, 1000),      # E = 1: tied optimal matchings (Hungarian path)
    "nginx_2ms": ("media_nginx_cal", 2, 120, 60.0, 2000),
}
# skip_synth.DAG_SHAPES at millisecond clocks: E = 4..8, several primary in-edges per callee
DAG_CASES = {f"{s}_ms": s for s in skip_synth.DAG_SHAPES}


def _batch(name):
    if name in DAG_CASES:
        return build_batch([skip_synth.dag_problem(DAG_CASES[name], 260, 20_000.0, seed=77, quantum=1000)[0]])
    shape, S, n, load, q = CASES[name]
    return build_batch_from_blocks([synth.make_block(shape, S, n, load, seed=77, quantum_us=q)])


def _check(name, backend):
    hb = _batch(name)
    ob, eb = tw_oracle.OracleBatch(hb), backend(hb)
    g = ob.params_pass0()
    o_sc, e_sc = ob.score(gauss=g), eb.score(gauss=g)
    # the input really has ties inside the kept lists: equal scores at neighbouring ranks
    s = o_sc["topk_score"]
    assert int((s[:, 1:] == s[:, :-1]).sum()) > 0, "no exact score ties in this input"
    for k in ("cut", "n_feasible", "topk_cnt", "topk_idx"):
        assert np.array_equal(e_sc[k], o_sc[k]), k
    assert np.array_equal(np.nan_to_num(e_sc["topk_score"]), np.nan_to_num(o_sc["topk_score"]))
    o_st, e_st = ob.stitch(o_sc["cut"], gauss=g), eb.stitch(o_sc["cut"], gauss=g)
    for k in ("assign", "mis_rank", "n_cand", "topk_idx", "topk_cnt"):
        assert np.array_equal(e_st[k], o_st[k]), k
    assert np.array_equal(e_st["counters"][:, :2], o_st["counters"][:, :2])


@pytest.mark.parametrize("name", list(CASES) + list(DAG_CASES))
def test_tie_order_is_the_references(name):
    _check(name, EmulBatch)


@pytest.mark.parametrize("name", list(CASES) + list(DAG_CASES))
def test_lane_parallel_tie_order_is_the_references(name):
    """Every in-span through the lane-parallel search (emul-combos): ties must go to the heap replay."""
    _check(name, partial(EmulBatch, light_combos=0))
