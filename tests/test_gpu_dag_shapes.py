"""GPU vs CPU oracle on two-pass services of five to eight callees and up to 28 score terms
(tests/skip_synth.DAG_SHAPES, the cases of tests/test_dag_shapes.py): k_score3 for E = 5..8 with its
packed per-in-span state, mixture records read in place for 17 and more terms, DAG masks on callees
4-7, callees with several primary in-edges summed in in_edges order, the stitch tiers, k_params0,
k_delays, k_assess and the refit.  Each pass is compared given the oracle's parameters: indices
exactly, scores to SCORE_TOL."""
import numpy as np
import pytest

from test_dag_shapes import CASES, oracle_run

pytestmark = pytest.mark.gpu

SCORE_TOL = 1e-9


@pytest.fixture(scope="module")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test needs a CUDA device")
    from traceweaver_b200.engine import Engine
    eng = Engine(0)
    yield eng
    eng.close()


def _np(t):
    return t.cpu().numpy()


def _dev(a, eng):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.int32)).to(eng.device)


def _max_diff(got, ref):
    """Largest |got - ref| where both are numbers; NaN must sit at the same places."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    return float(np.max(np.abs(got - ref), where=~np.isnan(ref), initial=0.0))


def _assert_same_bits(got, ref, what):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), what
    assert got[~nan].tobytes() == ref[~nan].tobytes(), what


# Mixture log-densities (pass 1) differ from the oracle's in the last bits (observed <= 6e-14 on an
# H100), so two tuples whose oracle scores tie exactly but are sums of DIFFERENT terms can come out one
# ulp apart on the device, and the heap order then keeps another member of the tie group.  Seen on
# k44-ms (28 terms, millisecond clocks): in-spans 86, 179 and 180.  Everywhere else pass-1 indices
# must be equal; there the reordered ranks must hold tuples the oracle scores as tied.
MIXTURE_TIE_ROWS = {"k44-ms": {86, 179, 180}}


def _assert_idx_equal_up_to_mixture_ties(got, ref, E, case):
    K = ref["topk_score"].shape[1]
    got, want = got.reshape(-1, K, E), ref["topk_idx"].reshape(-1, K, E)
    rows = set(np.flatnonzero((got != want).any(axis=(1, 2))).tolist())
    assert rows <= MIXTURE_TIE_ROWS.get(case, set()), f"pass-1 score: topk_idx differs on in-spans {sorted(rows)}"
    for i in rows:
        s = ref["topk_score"][i]
        for k in np.flatnonzero((got[i] != want[i]).any(axis=1)):
            tied = np.sum(s == s[k]) > 1 or k == K - 1    # rank K - 1 may tie with an unlisted tuple
            assert tied, (i, k, s.tolist())


def _path_row(eng, r, prm0, prm1):
    """(E, terms, tiles, redone tiles in pass 0, in pass 1, in-place mixture records) of one service."""
    E, nterm = r["prob"].E, len(r["prob"].terms())
    eng.score(prm0, want_used=True)
    tiles, redo0 = eng.tile_count(), eng.redo_tile_count()
    eng.score(prm1, want_used=True)
    redo1 = eng.redo_tile_count()
    return dict(E=E, terms=nterm, tiles=tiles, redo0=redo0, redo1=redo1, in_place=nterm > 16)


@pytest.mark.parametrize("case", CASES)
def test_each_pass_matches_oracle(engine, case):
    from oracle import tw_oracle
    r = oracle_run(case)
    hb, eng = r["hb"], engine
    ob = tw_oracle.OracleBatch(hb)
    eng.bind(hb)
    eng.prepare()
    # k_params0: mean and standard deviation bit for bit (NaN where a batch has too few samples)
    g_dev, g = _np(eng.params_pass0().table), r["gauss"]
    _assert_same_bits(g_dev[:, :2], g[:, :2], "params_pass0")
    assert _max_diff(g_dev[:, 2], g[:, 2]) <= 1e-12                  # log(sigma): device log()
    diffs = {}
    # pass 0 with the oracle's Gaussians
    prm = eng.params_from_host(gauss=g)
    sc = eng.score(prm, want_used=True)
    eng.status()
    o_sc = r["sc"]
    for k in ("cut", "n_feasible", "topk_cnt", "topk_idx"):
        assert np.array_equal(_np(sc[k]), o_sc[k]), f"pass-0 score: {k}"
    diffs["score0"] = _max_diff(_np(sc["topk_score"]), o_sc["topk_score"])
    o_st = r["st"]
    for und in (None, sc):                                   # search path and adopt / run paths
        for want_topk in (False, True):
            st = eng.stitch(prm, sc["cut"], undeleted=und, want_topk=want_topk)
            eng.status()
            what = f"pass-0 stitch (undeleted={und is not None}, want_topk={want_topk})"
            for k in ("assign", "mis_rank", "n_cand"):
                assert np.array_equal(_np(st[k]), o_st[k]), f"{what}: {k}"
            assert np.array_equal(_np(st["counters"])[:, :2], o_st["counters"][:, :2]), what
            if want_topk:
                assert np.array_equal(_np(st["topk_cnt"]), o_st["topk_cnt"]), what
                assert np.array_equal(_np(st["topk_idx"]), o_st["topk_idx"]), what
                diffs["stitch0"] = max(diffs.get("stitch0", 0.0), _max_diff(_np(st["topk_score"]), o_st["topk_score"]))
    # k_delays on the oracle's assignment: the refit's samples, bit for bit
    d, c = eng.delays(_dev(o_st["assign"], eng))
    od, oc = r["delays"]
    d, c = _np(d), _np(c)
    assert np.array_equal(c, oc)
    for o, n in zip(hb.term_sample_off[:-1], oc):
        assert d[o:o + n].tobytes() == od[o:o + n].tobytes()
    # pass 1 with the oracle's mixtures
    mix = r["mix"]
    prm1 = eng.params_from_host(mix=mix)
    sc1 = eng.score(prm1, want_used=True)
    eng.status()
    o_sc1 = r["sc1"]
    for k in ("cut", "n_feasible", "topk_cnt"):
        assert np.array_equal(_np(sc1[k]), o_sc1[k]), f"pass-1 score: {k}"
    diffs["score1"] = _max_diff(_np(sc1["topk_score"]), o_sc1["topk_score"])
    _assert_idx_equal_up_to_mixture_ties(_np(sc1["topk_idx"]), o_sc1, r["prob"].E, case)
    o_st1 = r["st1"]
    st1 = eng.stitch(prm1, sc["cut"], undeleted=sc1)
    eng.status()
    for k in ("assign", "mis_rank", "n_cand"):
        assert np.array_equal(_np(st1[k]), o_st1[k]), f"pass-1 stitch: {k}"
    assert np.array_equal(_np(st1["counters"])[:, :2], o_st1["counters"][:, :2])
    # k_assess: the truth and the final assignment under both passes' parameters
    for name, a in (("truth", r["truth"].reshape(-1)), ("final", o_st1["assign"])):
        for p, kw in ((prm, dict(gauss=g)), (prm1, dict(mix=mix))):
            lk, orc = eng.score_assignments(p, _dev(a, eng)), ob.score_assignments(a, **kw)
            assert np.array_equal(_np(lk["code"]), orc["code"]), name
            assert np.array_equal(_np(lk["prob_count"]), orc["prob_count"]), name
            key = f"assess-{name}"
            diffs[key] = max(diffs.get(key, 0.0), _max_diff(_np(lk["score"]), orc["score"]))
    print(f"\n{case}: max |score - oracle| " + " ".join(f"{k}={v:.3g}" for k, v in diffs.items()))
    assert max(diffs.values()) <= SCORE_TOL, diffs
    # pass-0 Gaussians: every case came out bit-equal on an H100, so that is what is asserted
    assert diffs["score0"] == 0.0 and diffs["stitch0"] == 0.0, diffs
    # k_score3 did the work: not every tile went to the sequential redo kernel
    row = _path_row(eng, r, prm, prm1)
    print(f"{case}: {row}")
    if row["E"] >= 5:
        assert row["redo0"] < row["tiles"] and row["redo1"] < row["tiles"], row


@pytest.mark.parametrize("case", [c for c in CASES if c.endswith("-us")])
def test_refit_matches_oracle(engine, case):
    """tw_gmm_refit on the oracle's pass-0 delays against the oracle's restated scikit-learn refit."""
    import torch
    from oracle import tw_oracle
    r = oracle_run(case)
    hb, eng = r["hb"], engine
    eng.bind(hb)
    eng.prepare()
    od, oc = r["delays"]
    prm, nsel = eng.gmm_refit(torch.from_numpy(od).to(eng.device), torch.from_numpy(oc).to(eng.device),
                              seed_select=10, want_selected=True)
    eng.status()
    # the terms of a service draw from one model-selection stream, one after the other (the oracle's
    # driver chains it the same way): term t starts after the draws of the terms before it
    _, _, max_n = tw_oracle.gmm_refit(hb.term_sample_off, od, oc, seed_select=10)
    draws = [tw_oracle.lib().two_gmm_draws_for(int(m)) for m in max_n]
    skip = np.concatenate([[0], np.cumsum(draws)[:-1]])
    omix, onsel, _ = tw_oracle.gmm_refit(hb.term_sample_off, od, oc, seed_select=10, rng_skip=skip)
    got = _np(prm.table)
    assert np.array_equal(_np(nsel), onsel)
    assert np.array_equal(got[:, 0], omix[:, 0])
    for t in range(len(omix)):
        k = int(omix[t, 0])
        w = 3 if k == 0 else k
        np.testing.assert_allclose(got[t, 1:1 + w], omix[t, 1:1 + w], rtol=1e-7, atol=1e-7)
        if k:
            np.testing.assert_allclose(got[t, 6:6 + k], omix[t, 6:6 + k], rtol=1e-7, atol=1e-7)
            np.testing.assert_allclose(got[t, 11:11 + k], omix[t, 11:11 + k], atol=1e-7)
            np.testing.assert_allclose(got[t, 16:16 + k], omix[t, 16:16 + k], atol=1e-7)


def test_whole_path_matches_oracle():
    """BatchSolver.solve (device refit included) against the oracle's whole path, microsecond clocks."""
    from oracle import tw_oracle
    from traceweaver_b200.api import BatchSolver
    from traceweaver_b200.batch import build_batch
    hb = build_batch([oracle_run(c)["prob"] for c in CASES if c.endswith("-us")])
    solver = BatchSolver(device=0, seed_select=10)
    out = {k: np.array(v) for k, v in solver.solve(hb).items()}
    solver.close()
    ref = tw_oracle.find_assignments(hb, 10, threads=4)
    assert np.array_equal(out["assign"], ref["assign"])
    assert np.array_equal(out["mis_rank"], ref["mis_rank"])
    assert np.array_equal(out["topk_idx"], ref["topk_idx"])
    assert np.array_equal(out["n_cand"], ref["n_cand_total"])
    assert np.array_equal(out["counters"][:, :2], ref["counters"][:, :2])


def test_paths_reached(engine):
    """Which device paths the cases reach: tiles k_score3 finished itself, tiles flagged for the
    sequential kernel, mixture records read in place (more than 16 terms)."""
    table = {}
    for case in CASES:
        r = oracle_run(case)
        engine.bind(r["hb"])
        engine.prepare()
        table[case] = _path_row(engine, r, engine.params_from_host(gauss=r["gauss"]),
                                engine.params_from_host(mix=r["mix"]))
    print("\ncase         E  terms  tiles  redo0  redo1  in-place")
    for case, row in table.items():
        print(f"{case:<12} {row['E']}  {row['terms']:>5}  {row['tiles']:>5}  {row['redo0']:>5}  {row['redo1']:>5}  "
              f"{row['in_place']}")
    for case, row in table.items():
        if row["E"] >= 5:
            assert row["redo0"] < row["tiles"] and row["redo1"] < row["tiles"], case
    # the 17- and 28-term microsecond services score pass 1 with mixture records read in place
    for terms in (17, 28):
        assert any(row["terms"] == terms and row["in_place"] and row["redo1"] < row["tiles"]
                   for case, row in table.items() if case.endswith("-us")), terms
    assert any(row["E"] == 8 and row["redo0"] > 0 for row in table.values())


def test_mixed_batch_equals_single_services():
    """Services of E = 1..8 and 2..28 terms in one batch (every per-E launch class, a stitch slab sized for
    E = 8): every service's results equal those of the service solved alone."""
    from traceweaver_b200 import _abi, synth
    from traceweaver_b200.api import BatchSolver
    from traceweaver_b200.batch import Problem, build_batch
    probs = []
    for k, shape in enumerate(("single", "hotel_search", "hotel_frontend", "media_nginx")):
        blk = synth.make_block(shape, 1, 260, 100.0, seed=60 + k)
        probs.append(Problem(in_start=blk.in_start[0], in_end=blk.in_end[0], out_start=[s[0] for s in blk.out_start],
                             out_end=[x[0] for x in blk.out_end], preds=blk.preds, name=shape))
    for c in ("dag5-us", "k33-ms", "mix7-us", "chain8-ms", "dag8-us", "k44-us", "diamond-ms"):
        probs.append(oracle_run(c)["prob"])
    hb = build_batch(probs)
    E = np.diff(hb.prob_ep_off)
    terms = np.diff(hb.ep_term_off[hb.prob_ep_off])
    assert set(E.tolist()) == set(range(1, 9)) and terms.min() == 2 and terms.max() == 28
    keys = ("assign", "mis_rank", "n_cand", "topk_idx", "topk_cnt", "counters")
    solver = BatchSolver(device=0, seed_select=10)
    whole = {k: np.array(v) for k, v in solver.solve(hb).items()}
    for p, prob in enumerate(probs):
        one = {k: np.array(v) for k, v in solver.solve(build_batch([prob])).items()}
        i0, i1 = int(hb.prob_in_off[p]), int(hb.prob_in_off[p + 1])
        t0, t1 = int(hb.prob_tuple_off[p]), int(hb.prob_tuple_off[p + 1])
        sl = dict(assign=slice(t0, t1), mis_rank=slice(i0, i1), n_cand=slice(i0, i1), topk_cnt=slice(i0, i1),
                  topk_idx=slice(_abi.TW_K * t0, _abi.TW_K * t1), counters=slice(p, p + 1))
        for k in keys:
            assert np.array_equal(whole[k][sl[k]], one[k]), (p, prob.name, k)
    solver.close()
