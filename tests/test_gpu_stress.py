"""GPU vs CPU oracle on synthetic services that exercise the edges the shipped traces do not:
heavy overlap (hundreds of candidate tuples per in-span, size-30 windows, candidates taken by
earlier windows), parallel DAGs with E = 4, single-endpoint services, tiny services, services too
large for the shared-memory taken bitmap, and candidate ranges wider than the narrow bitmaps.
Each pass is compared given the SAME parameters (the oracle's), so the comparison is bit-exact for
indices and 1e-9 for scores; the whole path (with the device refit) is compared on moderate loads."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test needs a CUDA device")
    from traceweaver_b200.engine import Engine
    eng = Engine(0)
    yield eng
    eng.close()


CASES = {
    # name: (shape, n_services, n_in, load)
    "hotel_overload": ("hotel_frontend", 6, 400, 600.0),     # ~7 concurrent requests: heavy windows
    "search_overload": ("hotel_search", 6, 400, 900.0),
    "nginx_parallel": ("media_nginx", 6, 300, 200.0),        # E = 4, no DAG edges
    "single_ep": ("single", 8, 300, 300.0),                  # E = 1 (bipartite case)
    "tiny": ("hotel_search", 16, 2, 100.0),                  # two in-spans: the minimum the reference accepts
    "big_service": ("hotel_frontend", 2, 5000, 100.0),       # taken bitmap in global memory
    "very_wide": ("single", 2, 300, 60000.0),                # > 64 candidates per in-span: wide bitmaps (score only)
    "wide_e2": ("hotel_search", 2, 300, 20000.0),            # E = 2, > 64 candidates on one callee: whole-warp redo (score only)
    # millisecond clocks: equal starts, exact score ties (heapq order, tests/test_ties.py) and tied
    # MWIS optima (TW_MWIS_TIE_TOL) are common
    "par3_ms": ("ali_par3", 4, 300, 60.0, 1000),
    "chain2_ms": ("ali_chain2", 4, 300, 100.0, 1000),
    "nginx_2ms": ("media_nginx_cal", 3, 200, 60.0, 2000),
    "leaf_dense_ms": ("ali_leaf", 4, 300, 300.0, 1000),      # E = 1: tied optimal matchings
}


def _batch(name):
    from traceweaver_b200 import synth
    from traceweaver_b200.batch import build_batch_from_blocks
    shape, S, n, load = CASES[name][:4]
    quantum = CASES[name][4] if len(CASES[name]) > 4 else 1
    blocks = [synth.make_block(shape, S, n, load, seed=123, quantum_us=quantum)]
    return blocks, build_batch_from_blocks(blocks)


def _np(t):
    return t.cpu().numpy()


@pytest.mark.parametrize("name", list(CASES))
def test_each_pass_matches_oracle(engine, name):
    from oracle import tw_oracle
    blocks, hb = _batch(name)
    ob = tw_oracle.OracleBatch(hb)
    eng = engine
    eng.bind(hb)
    eng.prepare()
    # pass-0 parameters: device vs oracle
    g_dev = _np(eng.params_pass0().table)
    g_cpu = ob.params_pass0()
    assert np.array_equal(np.nan_to_num(g_dev[:, :2], nan=-1.0), np.nan_to_num(g_cpu[:, :2], nan=-1.0))
    prm = eng.params_from_host(gauss=g_cpu)
    sc = eng.score(prm, want_used=True)
    o_sc = ob.score(gauss=g_cpu)
    eng.status()
    assert np.array_equal(_np(sc["cut"]), o_sc["cut"])
    assert np.array_equal(_np(sc["n_feasible"]), o_sc["n_feasible"])
    assert np.array_equal(_np(sc["topk_cnt"]), o_sc["topk_cnt"])
    assert np.array_equal(_np(sc["topk_idx"]), o_sc["topk_idx"])
    np.testing.assert_allclose(_np(sc["topk_score"]), o_sc["topk_score"], rtol=0, atol=1e-9, equal_nan=True)
    if name == "wide_e2":
        # flagged tiles hold in-spans with thousands of combinations over two callees: the redo kernel
        # scores them with the whole warp and marks the wide maps from several lanes at once.  Scoring
        # pass only: windows this dense exhaust the exact MWIS node budget (DESIGN.md §8).
        assert _np(sc["used_wide"]).max() == 1
        return
    if name == "very_wide":
        # ~100 interchangeable candidates per in-span: the candidate maps overflow the narrow bitmaps
        # (k_score<32,64> redo).  The stitch is not compared here: 31-in-span windows this dense
        # exhaust the exact MWIS node budget (DESIGN.md §8) in the engine and in the oracle alike.
        assert _np(sc["used_wide"]).max() == 1
        # E = 1: the engine solves these windows as exact bipartite matchings (Hungarian; checked
        # against scipy in tests/test_assignment.py), so it must finish within its budgets and
        # return a conflict-free assignment
        st = eng.stitch(prm, sc["cut"], undeleted=sc)
        eng.status()
        a = _np(st["assign"])
        for pidx in range(hb.n_problems):
            to, n = int(hb.prob_tuple_off[pidx]), int(hb.prob_in_off[pidx + 1] - hb.prob_in_off[pidx])
            col = a[to:to + n]
            used = col[col >= 0]
            assert len(np.unique(used)) == len(used)
            assert (col >= 0).mean() > 0.9
        return
    o_st = ob.stitch(o_sc["cut"], gauss=g_cpu)
    for und in (None, sc):                                   # search path and adopt / run paths
        st = eng.stitch(prm, sc["cut"], undeleted=und)
        eng.status()
        assert np.array_equal(_np(st["assign"]), o_st["assign"]), und is None
        assert np.array_equal(_np(st["mis_rank"]), o_st["mis_rank"])
        assert np.array_equal(_np(st["n_cand"]), o_st["n_cand"])
        assert np.array_equal(_np(st["counters"])[:, :2], o_st["counters"][:, :2])
    st = eng.stitch(prm, sc["cut"], want_topk=True)
    eng.status()
    assert np.array_equal(_np(st["topk_idx"]), o_st["topk_idx"])
    # pass 1 with the oracle's mixtures
    d, c = ob.delays(o_st["assign"])
    mix, _, _ = tw_oracle.gmm_refit(hb.term_sample_off, d, c, seed_select=10)
    prm1 = eng.params_from_host(mix=mix)
    sc1 = eng.score(prm1, want_used=True)
    o_sc1 = ob.score(mix=mix)
    assert np.array_equal(_np(sc1["topk_idx"]), o_sc1["topk_idx"])
    np.testing.assert_allclose(_np(sc1["topk_score"]), o_sc1["topk_score"], rtol=0, atol=1e-9, equal_nan=True)
    o_st1 = ob.stitch(o_sc["cut"], mix=mix)
    st1 = eng.stitch(prm1, sc["cut"], undeleted=sc1)
    eng.status()
    assert np.array_equal(_np(st1["assign"]), o_st1["assign"])
    assert np.array_equal(_np(st1["mis_rank"]), o_st1["mis_rank"])


# (the millisecond-clock cases are compared pass by pass above, with the oracle's mixtures: their delay
# samples hold a handful of distinct values, where the BIC arg-min of the refit is ill-conditioned —
# tests/gmm_conditioning.py — so a whole-path comparison would test summation order, not the engine)
@pytest.mark.parametrize("name", ["nginx_parallel", "single_ep", "tiny"])
def test_whole_path_matches_oracle(name):
    from oracle import tw_oracle
    from traceweaver_b200.api import BatchSolver
    blocks, hb = _batch(name)
    solver = BatchSolver(device=0, seed_select=10)
    out = solver.solve(hb)
    solver.close()
    ref = tw_oracle.find_assignments(hb, 10, threads=2)
    assert np.array_equal(out["assign"], ref["assign"])
    assert np.array_equal(out["topk_idx"], ref["topk_idx"])
    assert np.array_equal(out["n_cand"], ref["n_cand_total"])


def test_chunked_solver_matches_single_pass():
    """BatchSolver's copy/compute overlap (service groups on two streams) must not change anything."""
    from traceweaver_b200 import synth
    from traceweaver_b200.api import BatchSolver
    from traceweaver_b200.batch import build_batch_from_blocks
    hb = build_batch_from_blocks([synth.make_block("hotel_frontend", 7, 300, 150.0, seed=5),
                                  synth.make_block("hotel_search", 6, 200, 150.0, seed=6)])
    one = BatchSolver(device=0, seed_select=10, chunks=1)
    ref = {k: v.copy() for k, v in one.solve(hb).items()}
    one.close()
    many = BatchSolver(device=0, seed_select=10, chunks=3)
    many.MIN_CHUNK_IN_SPANS = 0
    for _ in range(2):                                       # second call re-uses the staging buffers
        got = many.solve(hb)
        for k in ref:
            assert np.array_equal(got[k], ref[k]), k
    assert many.last_chunks == 3
    # the caller refills its buffers in place: the next call must see the new contents
    hb2 = build_batch_from_blocks([synth.make_block("hotel_frontend", 7, 300, 150.0, seed=15),
                                   synth.make_block("hotel_search", 6, 200, 150.0, seed=16)])
    one = BatchSolver(device=0, seed_select=10, chunks=1)
    ref2 = {k: v.copy() for k, v in one.solve(hb2).items()}
    one.close()
    for name in ("in_start", "in_end", "out_start", "out_end"):
        hb.arrays[name][:] = hb2.arrays[name]
    got2 = many.solve(hb)
    for k in ref2:
        assert np.array_equal(got2[k], ref2[k]), k
    assert not np.array_equal(ref["assign"], ref2["assign"])
    # results of the previous call are still intact (two result sets alternate)
    for k in ref:
        assert np.array_equal(got[k], ref[k]), k
    many.close()


def test_engine_limits_fail_loudly(engine):
    """E > 8 is rejected at bind time with TW_ERR_INVALID, not mis-solved."""
    from traceweaver_b200 import _abi
    from traceweaver_b200.batch import Problem, build_batch
    s = np.arange(4, dtype=np.int64) * 1000
    p = Problem(in_start=s, in_end=s + 900, out_start=[s + 10] * 9, out_end=[s + 20] * 9, preds=[[]] * 9)
    with pytest.raises(ValueError):
        build_batch([p])
    hb = build_batch([p], validate=False)
    with pytest.raises(_abi.TwError) as ei:
        engine.bind(hb)
    assert ei.value.code == -1


def test_one_service_of_120k_spans_equals_oracle():
    """A single service with 30 000 incoming spans (120 000 spans, lists far beyond the 16 384 spans the
    shared-memory end-time sort takes): long lists are sorted in global memory (k_sort_ends_long), the
    stitch warp walks all windows, the refit fits 30 000 samples per term.  Engine == oracle."""
    import torch
    from oracle import tw_oracle
    from traceweaver_b200 import synth
    from traceweaver_b200.api import BatchSolver
    from traceweaver_b200.batch import build_batch_from_blocks
    blk = synth.make_block("hotel_frontend", 1, 30_000, 100.0, seed=3)
    hb = build_batch_from_blocks([blk])
    solver = BatchSolver(device=0, seed_select=10)
    out = solver.solve(hb)
    solver.close()
    ref = tw_oracle.find_assignments(hb, 10, threads=4)
    assert np.array_equal(out["assign"], ref["assign"])
    assert np.array_equal(out["mis_rank"], ref["mis_rank"])
    assert np.array_equal(out["topk_idx"], ref["topk_idx"])
    assert np.array_equal(out["counters"][:, :2], ref["counters"][:, :2])
    truth = synth.truth_assign([blk])
    assert (out["assign"] == truth).mean() > 0.99


def _engine_vs_profiler(eng, fn, trace):
    """(launch_count() delta, kernels of the library the CUDA profiler recorded) around fn()."""
    import json
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    l0 = eng.launch_count()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(str(trace))
    with open(trace) as f:
        events = json.load(f)["traceEvents"]
    seen = sum(1 for ev in events if ev.get("cat") == "kernel" and "tw::k_" in ev.get("name", ""))
    return eng.launch_count() - l0, seen


def test_launch_count_matches_profiler(engine, tmp_path):
    """launch_count() counts the kernels the engine issues, conditional launches included: a whole
    solve step, the global-memory sort of lists longer than 16 384 spans, accuracy without trace ids."""
    import torch
    from traceweaver_b200 import synth, truth
    from traceweaver_b200.batch import build_batch_from_blocks
    from traceweaver_b200.predictor import solve_bound
    engine.bind(build_batch_from_blocks(synth.hotel_stream(6, 200, seed=7)))
    counted, seen = _engine_vs_profiler(engine, lambda: solve_bound(engine), tmp_path / "solve.json")
    assert seen > 0 and counted == seen
    hb = build_batch_from_blocks([synth.make_block("hotel_frontend", 1, 20_000, 100.0, seed=3)])
    engine.bind(hb)
    counted, seen = _engine_vs_profiler(engine, engine.prepare, tmp_path / "prepare.json")
    assert counted == seen == 4                              # prev index, sort, long-list sort, tile windows
    tl = truth.TraceLists.from_host_batch(hb, None, 0)
    z = torch.zeros(int(hb.prob_tuple_off[-1]), dtype=torch.int32, device=engine.device)
    counted, seen = _engine_vs_profiler(engine, lambda: truth.accuracy(engine, tl, z, z), tmp_path / "accuracy.json")
    assert counted == seen == 2                              # no trace ids: no per-trace reduction
