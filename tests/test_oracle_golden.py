"""Pin the CPU oracle (oracle/tw_oracle.c) to the reference: every golden fixture was minted by
running the reference's own executor.py + TraceWeaverV3 in the build container
(tests/golden/make_goldens.py).  The same checks run on "emul": the engine's device functions
(traceweaver_b200/csrc/tw_core.cuh) compiled for the CPU and stepped thread by thread
(tests/emul/), because the build container has no GPU.  CPU only."""
from functools import partial

import numpy as np
import pytest

from golden_util import Golden, golden_files
from oracle import tw_oracle
from emul_backend import EmulBatch
from traceweaver_b200 import _abi
from traceweaver_b200.batch import build_batch

FILES = golden_files()
IDS = [f.split("/")[-1][:-4] for f in FILES]
SCORE_TOL = 1e-5   # north-star tolerance on log-likelihood scores


def test_goldens_present():
    assert len(FILES) >= 10


# Same device functions with the term tables disabled (per-leaf evaluation path)
EmulLazy = partial(EmulBatch, table_cap=0)
# Every in-span through the lane-parallel combination path + partial top-K merge
EmulCombos = partial(EmulBatch, light_combos=0)

BACKENDS = {"oracle": tw_oracle.OracleBatch, "emul": EmulBatch, "emul-lazy": EmulLazy, "emul-combos": EmulCombos}


@pytest.fixture(scope="module", params=[(f, b) for f in FILES for b in BACKENDS],
                ids=[f"{i}-{b}" for i in IDS for b in BACKENDS])
def case(request):
    path, backend = request.param
    g = Golden(path)
    prob = g.problem()
    hb = build_batch([prob])
    return g, prob, hb, BACKENDS[backend](hb)


def _idx_view(flat, n, E):
    return flat.reshape(n, _abi.TW_K, E)


def test_topological_layout(case):
    g, prob, hb, ob = case
    assert hb.no_skip()
    assert prob.E == len(g.topo)


def test_params_pass0_match_reference(case):
    """ComputeEpPairDistParams3 (v3:580-646): mean exact, std to 1e-12 relative."""
    g, prob, hb, ob = case
    want = g.gauss_table(prob)
    got = ob.params_pass0().reshape(want.shape)
    assert np.array_equal(got[..., 0], want[..., 0])
    np.testing.assert_allclose(got[..., 1], want[..., 1], rtol=1e-12, atol=0)


def test_windows_and_feasible_counts(case):
    """CreateWindows2 (v3:1020-1078)."""
    g, prob, hb, ob = case
    res = ob.score()
    assert tw_oracle.windows_from_cuts(res["cut"]) == g.windows()
    assert np.array_equal(res["n_feasible"], g.z["pre_cnt"])


@pytest.mark.parametrize("pass_id", [0, 1])
def test_topk_without_deletion(case, pass_id):
    """top_k_2 = FindTopKAssignments(K=5) on the undeleted lists (v3:1185)."""
    g, prob, hb, ob = case
    if pass_id == 0:
        res = ob.score(gauss=g.gauss_table(prob))
    else:
        res = ob.score(mix=g.mix_table(prob))
    n, E = prob.n_in, prob.E
    assert np.array_equal(res["topk_cnt"], g.z["topk2_cnt"][pass_id])
    want_s = g.z["topk2_score"][pass_id]
    np.testing.assert_allclose(res["topk_score"], want_s, rtol=0, atol=SCORE_TOL, equal_nan=True)
    assert np.array_equal(_idx_view(res["topk_idx"], n, E), g.z["topk2_idx"][pass_id])
    # tighter than the contract: the restatement follows scipy/sklearn operation order
    finite = np.isfinite(want_s)
    assert np.max(np.abs(res["topk_score"][finite] - want_s[finite])) < 1e-9


@pytest.mark.parametrize("pass_id", [0, 1])
def test_hot_loop_pass(case, pass_id):
    """top_k with deletion (v3:1182), MWIS per window (v3:1193), AddAssignment (v1:433-463)."""
    g, prob, hb, ob = case
    cut = ob.score()["cut"]
    kw = dict(gauss=g.gauss_table(prob)) if pass_id == 0 else dict(mix=g.mix_table(prob))
    res = ob.stitch(cut, **kw)
    n, E = prob.n_in, prob.E
    assert np.array_equal(res["topk_cnt"], g.z["topk_cnt"][pass_id])
    np.testing.assert_allclose(res["topk_score"], g.z["topk_score"][pass_id], rtol=0, atol=SCORE_TOL,
                               equal_nan=True)
    assert np.array_equal(_idx_view(res["topk_idx"], n, E), g.z["topk_idx"][pass_id])
    assert np.array_equal(res["mis_rank"], g.z["mis_rank"][pass_id])
    if pass_id == g.meta["passes"] - 1:
        assert np.array_equal(res["assign"].reshape(E, n), g.z["assign"])
        assert res["counters"][0, 0] == g.meta["not_best_count"]
        assert res["counters"][0, 1] == g.meta["cnt_unassigned"]


def test_candidate_counts_accumulate_over_passes(case):
    """per_span_candidates is not reset between iterations (v3:1093 vs :1159)."""
    g, prob, hb, ob = case
    cut = ob.score()["cut"]
    c0 = ob.stitch(cut, gauss=g.gauss_table(prob), want_topk=False)["n_cand"]
    c1 = ob.stitch(cut, mix=g.mix_table(prob), want_topk=False)["n_cand"]
    assert np.array_equal(c0.astype(np.int64) + c1, g.z["per_span_candidates"])


def test_delays_feed_the_refit(case):
    """durations of ComputeEpPairDistParams5 (v3:721-760): sample counts per term."""
    g, prob, hb, ob = case
    cut = ob.score()["cut"]
    a0 = ob.stitch(cut, gauss=g.gauss_table(prob), want_topk=False)["assign"]
    delays, counts = ob.delays(a0)
    mis0 = g.z["mis_rank"][0]
    assert np.all(counts == int((mis0 >= 0).sum()))
    assert np.all(np.isfinite(delays))
