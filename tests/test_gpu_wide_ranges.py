"""GPU vs CPU oracle on services whose candidate ranges leave the 64-bit maps of k_score3
(tests/wide_synth.py, the cases of tests/test_wide_ranges.py): the redo kernel k_score on ranges of 65 to
2048 spans (staged and unstaged slices, the carry-in helper over the global arrays, the term-table cap,
whole-warp combinations), k_cut's wide-prev branch, k_stitch_units' extent of wide in-spans, and the
stitch's search tier on wide ranges.  Each pass is compared given the oracle's parameters.  Also the
engine's two search limits: TW_ERR_RANGE_LIMIT at a feasible offset of 2048, and TW_ERR_MWIS_LIMIT with
BatchSolver.solve(strict=False)."""
import ctypes as C

import numpy as np
import pytest

import wide_synth as ws
from test_wide_ranges import CASES, SOLVED, oracle_run, problem

pytestmark = pytest.mark.gpu

SCORE_TOL = 1e-9


@pytest.fixture(scope="module")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test needs a CUDA device")
    from traceweaver_b200.engine import Engine
    eng = Engine(0)
    eng.lib.tw_debug_stitch_grid.argtypes = [C.c_void_p, C.c_int]
    eng.lib.tw_debug_node_limit.argtypes = [C.c_void_p, C.c_longlong]
    eng.lib.tw_debug_node_limit.restype = C.c_longlong
    yield eng
    eng.close()


def _np(t):
    return t.cpu().numpy()


def _max_diff(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    return float(np.max(np.abs(got - ref), where=~np.isnan(ref), initial=0.0))


def _assert_same_bits(got, ref, what):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), what
    assert got[~nan].tobytes() == ref[~nan].tobytes(), what


def _long_in_spans(name):
    return [L.pos for L in CASES[name].longs]


def _check_stitch(st, o_st, what, want_topk):
    for k in ("assign", "mis_rank", "n_cand"):
        assert np.array_equal(_np(st[k]), o_st[k]), f"{what}: {k}"
    assert np.array_equal(_np(st["counters"])[:, :2], o_st["counters"][:, :2]), f"{what}: counters"
    if want_topk:
        assert np.array_equal(_np(st["topk_cnt"]), o_st["topk_cnt"]), f"{what}: topk_cnt"
        assert np.array_equal(_np(st["topk_idx"]), o_st["topk_idx"]), f"{what}: topk_idx"
        return _max_diff(_np(st["topk_score"]), o_st["topk_score"])
    return 0.0


@pytest.mark.parametrize("name", SOLVED)
def test_each_pass_matches_oracle(engine, name):
    r = oracle_run(name)
    hb, eng = r["hb"], engine
    eng.bind(hb)
    eng.prepare()
    g_dev, g = _np(eng.params_pass0().table), r["gauss"]
    _assert_same_bits(g_dev[:, :2], g[:, :2], "params_pass0")        # mean and standard deviation
    assert _max_diff(g_dev[:, 2], g[:, 2]) <= 1e-12                  # log(sigma): device log()
    diffs = {}
    prm = eng.params_from_host(gauss=g)
    sc = eng.score(prm, want_used=True)
    eng.status()
    o_sc = r["sc"]
    for k in ("cut", "n_feasible", "topk_cnt", "topk_idx"):
        assert np.array_equal(_np(sc[k]), o_sc[k]), f"pass-0 score: {k}"
    diffs["score0"] = _max_diff(_np(sc["topk_score"]), o_sc["topk_score"])
    assert eng.redo_tile_count() >= len(ws.wide_tiles(r["prob"])) > 0
    wide = _np(sc["used_wide"])
    assert all(wide[i] == 1 for i in _long_in_spans(name))
    for und in (None, sc):                                   # whole services / units, search / run / adopt tiers
        for want_topk in (False, True):
            st = eng.stitch(prm, sc["cut"], undeleted=und, want_topk=want_topk)
            eng.status()
            d = _check_stitch(st, r["st"], f"pass-0 stitch (undeleted={und is not None}, want_topk={want_topk})",
                              want_topk)
            diffs["stitch0"] = max(diffs.get("stitch0", 0.0), d)
    prm1 = eng.params_from_host(mix=r["mix"])
    sc1 = eng.score(prm1, want_used=True)
    eng.status()
    o_sc1 = r["sc1"]
    for k in ("cut", "n_feasible", "topk_cnt", "topk_idx"):
        assert np.array_equal(_np(sc1[k]), o_sc1[k]), f"pass-1 score: {k}"
    diffs["score1"] = _max_diff(_np(sc1["topk_score"]), o_sc1["topk_score"])
    for und in (None, sc1):
        for want_topk in (False, True):
            st1 = eng.stitch(prm1, sc["cut"], undeleted=und, want_topk=want_topk)
            eng.status()
            d = _check_stitch(st1, r["st1"], f"pass-1 stitch (undeleted={und is not None}, want_topk={want_topk})",
                              want_topk)
            diffs["stitch1"] = max(diffs.get("stitch1", 0.0), d)
    print(f"\n{name}: max |score - oracle| " + " ".join(f"{k}={v:.3g}" for k, v in diffs.items()))
    assert diffs["score0"] == 0.0 and diffs["stitch0"] == 0.0, diffs      # pass 0: bit for bit
    assert max(diffs.values()) <= SCORE_TOL, diffs


@pytest.mark.parametrize("name", [k for k in SOLVED if CASES[k].clock == "us"])
def test_whole_path_matches_oracle(name):
    """BatchSolver.solve against the oracle.  Where the conditioning check of the refit (tests/gmm_cases.admit:
    the oracle's double and long double refits agree, no Lloyd ties, a clear BIC gap) admits every term of
    the oracle's pass-0 delays, the whole path must equal the oracle's.  Elsewhere most delay samples of a
    term hold one value (every short request has its children at the same offsets), the selected mixtures
    are not determined to the last bit, and the last pass is compared under the mixtures the call refitted:
    the oracle's pass 1 on them must give the call's top-K lists, assignment and counts."""
    import gmm_cases
    from oracle import tw_oracle
    from traceweaver_b200.api import BatchSolver
    r = oracle_run(name)
    hb = r["hb"]
    solver = BatchSolver(device=0, seed_select=10)
    out = {k: np.array(v) for k, v in solver.solve(hb, want_mixtures=True).items()}
    solver.close()
    ob = tw_oracle.OracleBatch(hb)
    d, c = ob.delays(r["st"]["assign"])
    admitted = bool(gmm_cases.admit(hb.term_sample_off, d, c)[0].all())
    if admitted:
        ref = tw_oracle.find_assignments(hb, 10, threads=4)
        ref_n_cand = ref["n_cand_total"]
    else:
        ref = dict(ob.score(mix=out["mixtures"]))
        st1 = ob.stitch(r["sc"]["cut"], mix=out["mixtures"])
        ref.update(assign=st1["assign"], mis_rank=st1["mis_rank"], counters=st1["counters"])
        ref_n_cand = r["st"]["n_cand"] + st1["n_cand"]
    print(f"\n{name}: refit conditioning admitted: {admitted}")
    for k in ("assign", "mis_rank", "topk_idx", "topk_cnt"):
        assert np.array_equal(out[k], ref[k]), k
    assert np.array_equal(out["n_cand"], ref_n_cand)
    assert np.array_equal(out["counters"][:, :2], ref["counters"][:, :2])


def test_strong_cut_next_to_wide_in_span(engine):
    """tests/wide_synth.strong_cut_case: the cut at Y is kept from being strong only by the wide in-span W's
    extent [lower_bound(start), upper_bound(end) - 1] in k_stitch_units.  Were it strong, Y and q would be
    stitched as a unit of their own, on a taken bitmap without W's choice, and q would take the span W took.
    Both passes, default grid and one block: equal to the oracle."""
    from test_wide_ranges import strong_cut_run
    r = strong_cut_run()
    eng, lib = engine, engine.lib
    eng.bind(r["hb"])
    eng.prepare()
    default_grid = lib.tw_debug_stitch_grid(eng.h, 0)
    try:
        for kw, o_sc, o_st in ((dict(gauss=r["gauss"]), r["sc"], r["st"]), (dict(mix=r["mix"]), r["sc1"], r["st1"])):
            prm = eng.params_from_host(**kw)
            sc = eng.score(prm, want_used=True)
            eng.status()
            for k in ("cut", "n_feasible", "topk_cnt", "topk_idx"):
                assert np.array_equal(_np(sc[k]), o_sc[k]), k
            assert _np(sc["used_wide"])[0] == 1
            for blocks in (default_grid, 1):
                assert lib.tw_debug_stitch_grid(eng.h, blocks) == blocks
                for und in (None, sc):
                    st = eng.stitch(prm, sc["cut"], undeleted=und)
                    eng.status()
                    _check_stitch(st, o_st, f"{list(kw)} {blocks} blocks undeleted={und is not None}", False)
    finally:
        lib.tw_debug_stitch_grid(eng.h, 0)


def test_unit_queue_one_block_grid(engine):
    """The service of many units (strong cuts before and after its long in-spans) on the default grid and
    on one block: both equal the oracle."""
    r = oracle_run("e1")
    eng, lib = engine, engine.lib
    eng.bind(r["hb"])
    eng.prepare()
    prm = eng.params_from_host(gauss=r["gauss"])
    sc = eng.score(prm, want_used=True)
    eng.status()
    default_grid = lib.tw_debug_stitch_grid(eng.h, 0)
    try:
        for blocks in (default_grid, 1):
            assert lib.tw_debug_stitch_grid(eng.h, blocks) == blocks
            st = eng.stitch(prm, sc["cut"], undeleted=sc)
            eng.status()
            _check_stitch(st, r["st"], f"{blocks} blocks", False)
    finally:
        lib.tw_debug_stitch_grid(eng.h, 0)


def _hotel_problems(k, seed):
    from traceweaver_b200 import synth
    from traceweaver_b200.batch import Problem
    out = []
    for j, shape in enumerate(("hotel_frontend", "hotel_search")[:k]):
        blk = synth.make_block(shape, 1, 260, 100.0, seed=seed + j)
        out.append(Problem(in_start=blk.in_start[0], in_end=blk.in_end[0], out_start=[s[0] for s in blk.out_start],
                           out_end=[x[0] for x in blk.out_end], preds=blk.preds, name=shape))
    return out


KEYS = ("assign", "mis_rank", "n_cand", "topk_idx", "topk_cnt", "counters")


def _slices(hb, p):
    from traceweaver_b200 import _abi
    i0, i1 = int(hb.prob_in_off[p]), int(hb.prob_in_off[p + 1])
    t0, t1 = int(hb.prob_tuple_off[p]), int(hb.prob_tuple_off[p + 1])
    return dict(assign=slice(t0, t1), mis_rank=slice(i0, i1), n_cand=slice(i0, i1), topk_cnt=slice(i0, i1),
                topk_idx=slice(_abi.TW_K * t0, _abi.TW_K * t1), counters=slice(p, p + 1))


def test_mixed_batch_equals_single_services():
    """Wide services beside ordinary hotel ones: every service's results equal those of it solved alone."""
    from traceweaver_b200.api import BatchSolver
    from traceweaver_b200.batch import build_batch
    probs = _hotel_problems(2, 70) + [problem(k) for k in ("e1-probe", "e2", "e5-par", "e2-ms")]
    hb = build_batch(probs)
    solver = BatchSolver(device=0, seed_select=10)
    whole = {k: np.array(v) for k, v in solver.solve(hb).items()}
    for p, prob in enumerate(probs):
        one = {k: np.array(v) for k, v in solver.solve(build_batch([prob])).items()}
        sl = _slices(hb, p)
        for k in KEYS:
            assert np.array_equal(whole[k][sl[k]], one[k]), (p, prob.name, k)
    solver.close()


def test_range_limit(engine):
    """Offset 2047 solves and equals the oracle; offset 2048 raises TW_ERR_RANGE_LIMIT with strict=True and
    with strict=False alike, and leaves no flag behind: the next batch equals the oracle."""
    from oracle import tw_oracle
    from traceweaver_b200 import _abi
    from traceweaver_b200.api import BatchSolver
    from traceweaver_b200.batch import build_batch
    solver = BatchSolver(device=0, seed_select=10)
    try:
        ok = build_batch([problem("e1-off2047")])
        out = solver.solve(ok)
        ref = tw_oracle.find_assignments(ok, 10, threads=4)
        assert np.array_equal(out["assign"], ref["assign"])
        bad = build_batch(_hotel_problems(1, 80) + [problem("e1-off2048")])
        for strict in (True, False):
            with pytest.raises(_abi.TwError) as ei:
                solver.solve(bad, strict=strict)
            assert ei.value.code == _abi.TW_ERR_RANGE_LIMIT
        nxt = build_batch(_hotel_problems(2, 90))
        out = solver.solve(nxt)
        ref = tw_oracle.find_assignments(nxt, 10, threads=4)
        assert np.array_equal(out["assign"], ref["assign"])
        assert np.array_equal(out["topk_idx"], ref["topk_idx"])
    finally:
        solver.close()
    # the engine-level score reports it too, and the flag is reset by the status call that raised it
    hb = build_batch([problem("e1-off2048")])
    g = tw_oracle.OracleBatch(hb).params_pass0()
    engine.bind(hb)
    engine.prepare()
    engine.score(engine.params_from_host(gauss=g), want_used=True)
    with pytest.raises(_abi.TwError) as ei:
        engine.status()
    assert ei.value.code == _abi.TW_ERR_RANGE_LIMIT
    engine.status()


def _set_limit(eng, n):
    return eng.lib.tw_debug_node_limit(eng.h, n)


def _stitch_limited(eng, hb, gauss, limit, units):
    """Pass-0 stitch of `hb` under the oracle's Gaussians at node limit `limit` (0: default), in units
    between strong cuts or (units=False, no undeleted lists) one unit per service; returns host arrays,
    the status code and the cut flags."""
    from traceweaver_b200 import _abi
    eng.bind(hb)
    eng.prepare()
    prm = eng.params_from_host(gauss=gauss)
    sc = eng.score(prm, want_used=True)
    eng.status()
    assert _set_limit(eng, limit) == (limit if limit > 0 else 2_000_000)
    st = eng.stitch(prm, sc["cut"], undeleted=sc if units else None)
    code = 0
    try:
        eng.status()
    except _abi.TwError as ex:
        code = ex.code
    return {k: _np(st[k]) for k in ("assign", "mis_rank", "n_cand", "counters")}, code, _np(sc["cut"])


def _threshold(run, hi):
    """The smallest node limit in [1, hi] at which run(limit) reports no failure: the largest node count of
    a window the limit applies to (windows of more than kSmallWindow in-spans; counters[:, 2] also holds the
    leaf counts of the small-window search, which takes no limit)."""
    lo = 1
    while lo < hi:
        mid = (lo + hi) // 2
        if run(mid):
            hi = mid
        else:
            lo = mid + 1
    return lo


def _two_blocks(synth, Problem):
    """One hotel_search service: a dense stretch (about 20 000 nodes in its largest window on the CPU build,
    beyond the plain search's budget, so the priced search and its node limit apply), a quiet gap, then a
    light stretch.  The gap is a strong cut with hundreds of in-spans after it: a later stitch unit."""
    a = synth.make_block("hotel_search", 1, 300, 6000.0, seed=124)
    b = synth.make_block("hotel_search", 1, 200, 100.0, seed=125)
    shift = int(max(a.in_end[0].max(), max(x[0].max() for x in a.out_end))) + 10_000_000
    cat = lambda x, y: np.concatenate([x, y + shift])
    return Problem(in_start=cat(a.in_start[0], b.in_start[0]), in_end=cat(a.in_end[0], b.in_end[0]),
                   out_start=[cat(x[0], y[0]) for x, y in zip(a.out_start, b.out_start)],
                   out_end=[cat(x[0], y[0]) for x, y in zip(a.out_end, b.out_end)], preds=a.preds, name="two_blocks")


def _pass1_code(eng, hb, mix, limit):
    """Status of the last pass alone (pass-1 score, stitch with its undeleted lists) under `mix` at `limit`."""
    from traceweaver_b200 import _abi
    eng.bind(hb)
    eng.prepare()
    prm1 = eng.params_from_host(mix=mix)
    top = eng.score(prm1, want_used=True)
    eng.status()
    _set_limit(eng, limit)
    try:
        eng.stitch(prm1, top["cut"], undeleted=top)
        eng.status()
        return 0
    except _abi.TwError as ex:
        return ex.code
    finally:
        _set_limit(eng, 0)


def test_node_limit_and_strict_false(engine):
    """TW_ERR_MWIS_LIMIT just below the largest window search of a batch.  Within the failed service, the
    in-spans before the failing window keep their results; from the failing window to the end of its stitch
    unit (the next strong cut) they stay unassigned, and the service's later units are solved as without
    the limit.  A service stitched as one unit is therefore unassigned from the failing window on.  Other
    services are untouched; solve(strict=False) reports exactly the failed service, strict=True raises, and
    a service whose first pass alone hit the limit is reported too."""
    from oracle import tw_oracle
    from traceweaver_b200 import _abi, synth
    from traceweaver_b200.api import BatchSolver
    from traceweaver_b200.batch import Problem, build_batch
    eng = engine
    blk = synth.make_block("hotel_frontend", 1, 300, 600.0, seed=123)
    probs = [problem("e2"), Problem(in_start=blk.in_start[0], in_end=blk.in_end[0],
                                    out_start=[x[0] for x in blk.out_start], out_end=[x[0] for x in blk.out_end],
                                    preds=blk.preds, name="hotel_frontend"), _two_blocks(synth, Problem)]
    P = 2
    hb = build_batch(probs)
    g = tw_oracle.OracleBatch(hb).params_pass0()
    thresholds = {}
    try:
        for units in (False, True):     # one unit per service (no undeleted lists), units between strong cuts
            full, code, cut = _stitch_limited(eng, hb, g, 0, units)
            assert code == 0
            thresholds[units] = _threshold(lambda n: _stitch_limited(eng, hb, g, n, units)[1] == 0,
                                           int(full["counters"][:, 2].max()))
            limit = thresholds[units] - 1
            assert limit > 0, "no window of the batch reaches the priced search"
            got, code, _ = _stitch_limited(eng, hb, g, limit, units)
            assert code == _abi.TW_ERR_MWIS_LIMIT
            assert np.flatnonzero(got["counters"][:, 3] != 0).tolist() == [P]
            assert got["counters"][P, 3] == _abi.TW_ERR_MWIS_LIMIT
            for p in range(P):                               # other services: as without the limit
                s = _slices(hb, p)
                for k in ("assign", "mis_rank", "n_cand"):
                    assert np.array_equal(got[k][s[k]], full[k][s[k]]), (p, k)
            sl = _slices(hb, P)
            n, E = probs[P].n_in, probs[P].E
            a_full = full["assign"][sl["assign"]].reshape(E, n)
            a_got = got["assign"][sl["assign"]].reshape(E, n)
            r_full, r_got = full["mis_rank"][sl["mis_rank"]], got["mis_rank"][sl["mis_rank"]]
            diff = np.flatnonzero((a_full != a_got).any(0) | (r_full != r_got))
            assert len(diff) > 0
            f = int(diff[0])                                 # first in-span of the failing window
            assert (a_got[:, :f] == a_full[:, :f]).all() and (r_got[:f] == r_full[:f]).all()
            rest = np.flatnonzero((a_got[:, f:] >= 0).any(0) | (r_got[f:] >= 0))
            u = f + int(rest[0]) if len(rest) else n         # first in-span assigned again
            assert (a_got[:, f:u] == -1).all() and (r_got[f:u] == -1).all()
            assert (a_got[:, u:] == a_full[:, u:]).all() and (r_got[u:] == r_full[u:]).all()
            c = cut[sl["mis_rank"]]
            print(f"\n{probs[P].name} units={units}: node limit {limit}, failing window at in-span {f}, "
                  f"unassigned up to {u} of {n}, assigned after it: {int((r_got[u:] >= 0).sum())}")
            if not units:
                assert u == n
            else:                                            # the later units are solved: the light stretch
                assert f < u < n and c[u] == 1 and (r_got[u:] >= 0).sum() > 100
    finally:
        _set_limit(eng, 0)
    # the whole path
    solver = BatchSolver(device=0, seed_select=10)
    try:
        ref = {k: np.array(v) for k, v in solver.solve(hb, want_mixtures=True).items()}

        def ok(n):
            for e in solver._engines:
                _set_limit(e, n)
            return len(solver.solve(hb, strict=False)["failed_services"]) == 0
        limit = _threshold(ok, int(ref["counters"][:, 2].max())) - 1
        assert limit > 0, "no window of the batch reaches the priced search"
        for e in solver._engines:
            _set_limit(e, limit)
        with pytest.raises(_abi.TwError) as ei:
            solver.solve(hb)
        assert ei.value.code == _abi.TW_ERR_MWIS_LIMIT
        out = solver.solve(hb, strict=False)
        assert out["failed_services"].tolist() == [P]
        assert out["counters"][P, 3] == _abi.TW_ERR_MWIS_LIMIT
        for p in range(P):
            assert out["counters"][p, 3] == 0
            s = _slices(hb, p)
            for k in KEYS:
                assert np.array_equal(out[k][s[k]], ref[k][s[k]]), (p, k)
        # a first-pass failure the last pass does not repeat: just below the first pass's threshold (the
        # engine-level run above, with the same Gaussians and undeleted lists), the last pass under the
        # mixtures the call refitted finishes, and the service is still reported
        lim0 = thresholds[True] - 1
        for e in solver._engines:
            _set_limit(e, lim0)
        out = {k: np.array(v) for k, v in solver.solve(hb, strict=False, want_mixtures=True).items()}
        for e in solver._engines:
            _set_limit(e, 0)
        code1 = _pass1_code(eng, hb, out["mixtures"], lim0)
        print(f"first-pass limit {lim0}: last pass alone -> {_abi.STATUS[code1]}, reported {out['failed_services']}")
        assert code1 == 0
        assert out["failed_services"].tolist() == [P] and out["counters"][P, 3] == _abi.TW_ERR_MWIS_LIMIT
    finally:
        for e in solver._engines:
            _set_limit(e, 0)
        solver.close()


def test_paths_reached(engine):
    """For each case: from the generated arrays (host), the widest feasible offset, whether the redo tile of
    its widest in-span stages its slice and the strong cuts under the device's cut flags; from the device,
    the tiles, the tiles it redid and the in-spans it marked wide."""
    rows = {}
    for name in SOLVED:
        r = oracle_run(name)
        prob = r["prob"]
        engine.bind(r["hb"])
        engine.prepare()
        sc = engine.score(engine.params_from_host(gauss=r["gauss"]), want_used=True)
        engine.status()
        ed = ws.edges(prob)
        i = int(np.argmax(ed["off"].max(1)))
        slc = [s for s in ed["slices"] if s[0] <= i < s[1]][0]
        rows[name] = dict(E=prob.E, C=int(ed["r"][i].max()), off=int(ed["off"][i].max()),
                          staged=slc[2] <= ws.STAGE_SPANS, tiles=engine.tile_count(), redo=engine.redo_tile_count(),
                          wide=int(_np(sc["used_wide"]).sum()),
                          strong=len(ws.strong_cuts(prob, _np(sc["cut"]))))
    print("\n             host                                  device")
    print("case         E     C   offset  staged  strong-cuts  tiles  redo  wide-in-spans")
    for name, w in rows.items():
        print(f"{name:<12} {w['E']}  {w['C']:>5}  {w['off']:>6}  {str(w['staged']):<6}  {w['strong']:>11}  "
              f"{w['tiles']:>5}  {w['redo']:>4}  {w['wide']:>13}")
    assert not rows["e1-c1537"]["staged"] and rows["e1-c1536"]["staged"]
    # the probe's second tile is not redone: k_cut decided its first in-span's flag against a wide prev
    assert rows["e1-probe"]["redo"] == len(ws.wide_tiles(problem("e1-probe")))
    assert rows["e1"]["strong"] > 10
