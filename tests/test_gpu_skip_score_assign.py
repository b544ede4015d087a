"""GPU: tw_skip_score_assignments — the score of a given assignment of a cache-mode service on the device.
Listed top-K tuples bit for bit, the engine's own final assignment and the golden truth against the skip
oracle's checker, reproducible service sums, that want_likelihood=False changes nothing, and the drop-in
predictor's last_likelihood in both regimes."""
import glob
import os

import numpy as np
import pytest

from assess.skip_oracle_assess import assess_service
from golden_util import Golden
from test_skip_mode import CACHE_DIR, FILES, IDS
from test_skip_score_assign import host_margin, rank_tuples, truth_with_skips
from traceweaver_b200 import skipmode

pytestmark = pytest.mark.gpu
K = 5
RTOL = 1e-12
RESULTS = ("assign", "mis_rank", "n_cand", "counters", "topk_score", "topk_idx", "topk_cnt", "top2_score", "top2_idx",
           "top2_cnt", "cut")


@pytest.fixture(scope="module")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test needs a CUDA device")
    from traceweaver_b200.engine import Engine
    eng = Engine(0)
    yield eng
    eng.close()


def _solve(eng, g, **kw):
    prob = g.problem()
    st = skipmode.SkipState()
    st.time_windows = [tuple(w) for w in g.meta["time_windows_before"]]
    return prob, skipmode.solve(eng, prob.in_start, prob.in_end, prob.out_start, prob.out_end, prob.preds,
                                labels=[g.meta["in_ep"]] + g.topo, state=st, **kw)


def _score(eng, prob, assign, res):
    return skipmode.score(eng, prob.in_start, prob.in_end, prob.out_start, prob.out_end, prob.preds, assign, res)


def _oracle(prob, res, assign):
    return assess_service(prob.in_start, prob.in_end, prob.out_start, prob.out_end, prob.preds, assign,
                          res["pair_params"], any(b > 0 for b in res["skip_budget"]))


@pytest.mark.parametrize("path", FILES, ids=IDS)
def test_listed_tuples_score_bit_identical(engine, path):
    """Every tuple of the engine's with-deletion (topk) and no-deletion (top2) lists scores its listed score
    bit for bit, with code 0."""
    prob, res = _solve(engine, Golden(path))
    for which in ("topk", "top2"):
        idx, cnt, score = res[f"{which}_idx"], res[f"{which}_cnt"], res[f"{which}_score"]
        for r in range(K):
            live = cnt > r
            if not live.any():
                break
            lk = _score(engine, prob, rank_tuples(idx, cnt, r), res)
            assert np.all(lk["code"][live] == 0) and np.all(lk["code"][~live] == 1)
            assert lk["score"][live].tobytes() == score[live, r].tobytes(), (which, r)


@pytest.mark.parametrize("path", FILES, ids=IDS)
def test_final_assignment_and_truth(engine, path):
    """want_likelihood=True: the engine's final assignment is unassigned (code 1) exactly cnt_unassigned
    times, its scores equal the oracle checker's, its margins follow their definition against top2; the
    golden truth scores and codes as the oracle checker says; the service sum is reproducible."""
    g = Golden(path)
    prob, res = _solve(engine, g, want_likelihood=True)
    code, score = res["chosen_code"], res["chosen_score"]
    assert int((code == 1).sum()) == int(res["counters"][0, 1])
    orc = _oracle(prob, res, res["assign"])
    assert np.array_equal(code, orc["code"])
    assert np.array_equal(res["service_codes"], orc["service_codes"])
    ok = code == 0
    assert np.allclose(score[ok], orc["score"][ok], rtol=RTOL, atol=0) and np.all(np.isnan(score[~ok]))
    m = host_margin(score, code, res["assign"], res["top2_score"], res["top2_idx"], res["top2_cnt"])
    assert np.array_equal(res["margin"], m, equal_nan=True)
    assert res["service_score"] == pytest.approx(score[ok].sum(), rel=1e-12)
    # the same assignment through score(): the same bits
    again = _score(engine, prob, res["assign"], res)
    for a, b in (("chosen_score", "score"), ("chosen_code", "code"), ("margin", "margin")):
        assert res[a].tobytes() == again[b].tobytes(), a
    assert np.float64(res["service_score"]).tobytes() == np.float64(again["service_score"]).tobytes()
    # the truth, the cached call as a skip span
    t = truth_with_skips(g, prob)
    lk = _score(engine, prob, t, res)
    orc = _oracle(prob, res, t)
    assert np.array_equal(lk["code"], orc["code"])
    ok = orc["code"] == 0
    assert ok.sum() > 0.5 * prob.n_in
    assert np.allclose(lk["score"][ok], orc["score"][ok], rtol=RTOL, atol=0)
    # reproducible: a second solve gives the same service sum, bit for bit
    _, res2 = _solve(engine, g, want_likelihood=True)
    assert np.float64(res2["service_score"]).tobytes() == np.float64(res["service_score"]).tobytes()


def test_default_off_changes_nothing(engine):
    """want_likelihood=False: every output and the launch count are those of a plain solve; True adds the
    two assessment launches and changes no other output."""
    g = Golden(FILES[0])
    eng = engine
    c0 = eng.launch_count()
    _, a = _solve(eng, g)
    c1 = eng.launch_count()
    _, b = _solve(eng, g, want_likelihood=True)
    c2 = eng.launch_count()
    _, c = _solve(eng, g)
    c3 = eng.launch_count()
    assert c2 - c1 == c1 - c0 + 2
    assert c3 - c2 == c1 - c0
    assert set(c) == set(a) and "chosen_score" not in a
    for k in RESULTS:
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() == np.asarray(c[k]).tobytes(), k
    for k in ("time_windows", "skip_budget", "large_delay"):
        assert a[k] == b[k] == c[k], k
    for k in ("skip_count", "pair_params"):
        assert np.array_equal(a[k], b[k], equal_nan=True) and np.array_equal(a[k], c[k], equal_nan=True), k


def _same(lk, iids, score, code, margin):
    got = np.array([lk["in_spans"][i] for i in iids])
    assert got[:, 1].astype(int).tolist() == np.asarray(code).astype(int).tolist()
    assert got[:, 0].tobytes() == np.asarray(score, np.float64).tobytes()
    assert got[:, 2].tobytes() == np.asarray(margin, np.float64).tobytes()


def test_predictor_likelihood_in_both_regimes():
    """The sequence of a cache-mode run (frontend with skip budgets, then search without) through ONE
    TraceWeaverV3(want_likelihood=True): the 6-tuples equal want_likelihood=False's, and last_likelihood
    equals skipmode.solve(want_likelihood=True) for the skip service and BatchSolver.solve(want_likelihood=True)
    for the two-pass one."""
    from test_gpu_pipeline import reference_call_args
    from traceweaver_b200 import refit
    from traceweaver_b200.api import BatchSolver
    from traceweaver_b200.batch import build_batch
    from traceweaver_b200.engine import Engine
    from traceweaver_b200.predictor import TraceWeaverV3
    files = sorted(glob.glob(os.path.join(CACHE_DIR, "hotel_load150_cache20__*.npz")))
    gs = {Golden(f).meta["process"]: Golden(f) for f in files}
    on, off = TraceWeaverV3({}, {}, device=0, want_likelihood=True), TraceWeaverV3({}, {}, device=0)
    eng, solver = Engine(0), BatchSolver(device=0, seed_select=10)
    try:
        for process in ("frontend", "search"):
            g = gs[process]
            in_parts, out_parts, truth, G = reference_call_args(g)
            args = ("MaxScoreBatchSubsetWithSkips", process, in_parts, out_parts, False, [], truth, G)
            c0, o0 = off.engine.launch_count(), on.engine.launch_count()
            want = off.FindAssignments(*args)
            got = on.FindAssignments(*args)
            c1, o1 = off.engine.launch_count(), on.engine.launch_count()
            assert got == want, process
            assert off.last_likelihood is None
            assert o1 - o0 == c1 - c0 + 2, process
            lk = on.last_likelihood
            in_ep, in_spans = list(in_parts.items())[0]
            in_spans = sorted(in_spans, key=lambda x: float(x.start_mus))
            iids = [s.GetId() for s in in_spans]
            assert set(lk["in_spans"]) == set(iids)
            if process == "frontend":
                assert lk["regime"] == "skip"
                _, ref = _solve(eng, g, want_topk=False, want_likelihood=True)
                _same(lk, iids, ref["chosen_score"], ref["chosen_code"], ref["margin"])
                assert np.float64(lk["service_score"]).tobytes() == np.float64(ref["service_score"]).tobytes()
                assert np.array_equal(lk["service_codes"], ref["service_codes"])
                continue
            assert lk["regime"] == "two_pass"
            # the batch, truth and term order the predictor hands the two-pass path
            parts = {ep: sorted(p, key=lambda x: float(x.start_mus)) for ep, p in out_parts.items()}
            prob, out_eps, _, out_ids = on._marshal(process, in_spans, parts, G, False)
            tr = np.full((prob.E, prob.n_in), -1, np.int32)
            for e, ep in enumerate(out_eps):
                lut = {sid: j for j, sid in enumerate(out_ids[e])}
                tr[e] = [lut.get(truth.get(ep, {}).get(i), -1) for i in iids]
            order = np.asarray(refit.reference_term_order(prob, [out_eps.index(ep) for ep in out_parts]), np.int32)
            ref = solver.solve(build_batch([prob]), truth_assign=tr.reshape(-1), term_order=order, want_likelihood=True)
            _same(lk, iids, ref["chosen_score"], ref["chosen_code"], ref["margin"])
            assert np.float64(lk["service_score"]).tobytes() == ref["service_loglik"][0].tobytes()
            assert np.array_equal(lk["service_codes"], ref["service_codes"][0])
    finally:
        eng.close()
        solver.close()
