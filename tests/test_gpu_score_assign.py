"""GPU: tw_score_assignments — the likelihood of a given assignment on the device.  Scores of top-K tuples
bit for bit, golden tuples and the truth against the goldens and the oracle, the per-in-span outputs of
BatchSolver.solve(want_likelihood=True), float64 binds, and that the new outputs change nothing else."""
import numpy as np
import pytest

from float_times_util import SOLVABLE, compress
from golden_util import Golden, golden_files
from assess_backends import oracle_score
from test_score_assign import host_margin, rank_assign

pytestmark = pytest.mark.gpu
FILES = golden_files(gpu=True)
K = 5
RESULTS = ("assign", "topk_idx", "topk_cnt", "n_cand", "counters", "mis_rank", "topk_score")
LIKELIHOOD = ("chosen_score", "chosen_code", "margin", "service_loglik", "service_codes", "mixtures", "mixture_off")
TOL = 1e-10


@pytest.fixture(scope="module")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test needs a CUDA device")
    from traceweaver_b200.engine import Engine
    eng = Engine(0)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def solver(engine):
    from traceweaver_b200.api import BatchSolver
    s = BatchSolver(device=0, seed_select=10)
    yield s
    s.close()


@pytest.fixture(scope="module")
def goldens():
    return [Golden(f) for f in FILES]


@pytest.fixture(scope="module")
def golden_batch(goldens):
    from traceweaver_b200.batch import build_batch
    probs = [g.problem() for g in goldens]
    hb = build_batch(probs)
    gauss = np.concatenate([g.gauss_table(p).reshape(-1, 3) for g, p in zip(goldens, probs)])
    mix = np.concatenate([g.mix_table(p) for g, p in zip(goldens, probs)])
    truth = np.concatenate([g.z["truth"].astype(np.int32).reshape(-1) for g in goldens])
    return hb, probs, gauss, mix, truth


def _np(t):
    return t.cpu().numpy()


def _dev(a, eng):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)


def _rank_assign_batch(hb, idx_flat, cnt, r):
    """Rank-r tuples of a batch's top-K lists (topk_idx layout) in the assign layout, -1 past the count."""
    out = np.empty(int(hb.prob_tuple_off[-1]), np.int32)
    for p in range(hb.n_problems):
        i0, i1 = int(hb.prob_in_off[p]), int(hb.prob_in_off[p + 1])
        t0, t1 = int(hb.prob_tuple_off[p]), int(hb.prob_tuple_off[p + 1])
        n, E = i1 - i0, (t1 - t0) // (i1 - i0)
        out[t0:t1] = rank_assign(idx_flat[K * t0:K * t1].reshape(n, K, E), cnt[i0:i1], r)
    return out


def _synthetic_batches():
    from traceweaver_b200 import synth
    from traceweaver_b200.batch import build_batch, build_batch_from_blocks
    return {
        "hotel": build_batch_from_blocks(synth.hotel_stream(24, 300, seed=3)),
        "media": build_batch_from_blocks(synth.media_stream(36, 300, seed=4)),
        "alibaba": build_batch_from_blocks(synth.alibaba_stream(36, 300, seed=5)),
        "shapes": build_batch_from_blocks([synth.make_block(s, 2, 260, 100.0, seed=40 + k)
                                           for k, s in enumerate(sorted(synth.SHAPES))]),
        "wide": build_batch([_wide(E, 230, seed=E * 10 + r) for E in range(5, 9) for r in range(2)]),
    }


def _wide(E, n, seed):
    """A service with E = 5..8 callees: odd callees follow the one before them (a DAG edge), even ones
    start off the in-span."""
    from traceweaver_b200.batch import Problem
    rng = np.random.default_rng(seed)
    in_s = 10**9 + np.cumsum(rng.integers(20, 200, n)).astype(np.int64)
    starts, ends, preds, last = [], [], [], in_s
    for e in range(E):
        base = ends[-1] if e % 2 else in_s
        st = base + rng.integers(1, 40, n)
        en = st + rng.integers(5, 120, n)
        starts.append(st)
        ends.append(en)
        preds.append([e - 1] if e % 2 else [])
        last = np.maximum(last, en)
    in_e = last + rng.integers(1, 30, n)
    out_s, out_e = [], []
    for st, en in zip(starts, ends):
        o = np.lexsort((en, st))
        out_s.append(st[o])
        out_e.append(en[o])
    return Problem(in_start=in_s, in_end=in_e, out_start=out_s, out_end=out_e, preds=preds, name=f"wide{E}")


@pytest.fixture(scope="module")
def batches(golden_batch):
    d = _synthetic_batches()
    d["goldens"] = golden_batch[0]
    return d


def _check_ranks(eng, prm, top, hb):
    """Every rank of a top-K list scored under the list's own params: the listed score, bit for bit."""
    idx, cnt, score = _np(top["topk_idx"]), _np(top["topk_cnt"]), _np(top["topk_score"])
    for r in range(K):
        live = cnt > r
        if not live.any():
            break
        lk = eng.score_assignments(prm, _dev(_rank_assign_batch(hb, idx, cnt, r), eng))
        code, got = _np(lk["code"]), _np(lk["score"])
        assert np.all(code[live] == 0) and np.all(code[~live] == 1)
        assert got[live].tobytes() == score[live, r].tobytes(), f"rank {r}"


@pytest.mark.parametrize("name", ["goldens", "hotel", "media", "alibaba", "shapes", "wide"])
def test_topk_tuples_score_bit_identical(engine, batches, name):
    from traceweaver_b200.predictor import solve_bound
    eng, hb = engine, batches[name]
    eng.bind(hb)
    res = solve_bound(eng, seed_select=10)
    top = dict(topk_idx=res["topk_idx"], topk_cnt=res["topk_cnt"], topk_score=res["topk_score"])
    _check_ranks(eng, res["params_pass1"], top, hb)
    # pass 0: the first tw_score_topk of the path, scored under the pass-0 records
    eng.prepare()
    p0 = eng.params_pass0()
    sc = eng.score(p0, want_used=True)
    _check_ranks(eng, p0, sc, hb)
    eng.status()


def test_golden_tuples_and_truth(engine, golden_batch):
    hb, probs, gauss, mix, truth = golden_batch
    eng = engine
    eng.bind(hb)
    for pid, (prm, kw) in enumerate(((eng.params_from_host(gauss=gauss), dict(gauss=gauss)),
                                     (eng.params_from_host(mix=mix), dict(mix=mix)))):
        idx = np.concatenate([Golden(f).z["topk2_idx"][pid].astype(np.int32).reshape(-1) for f in FILES])
        cnt = np.concatenate([Golden(f).z["topk2_cnt"][pid] for f in FILES])
        want = np.concatenate([Golden(f).z["topk2_score"][pid] for f in FILES])
        for r in range(K):
            a = _rank_assign_batch(hb, idx, cnt, r)
            got = eng.score_assignments(prm, _dev(a, eng))
            orc = oracle_score(hb, a, **kw)
            live = cnt > r
            g, ref = _np(got["score"])[live], want[live, r]
            assert np.array_equal(_np(got["code"]), orc["code"])
            assert np.array_equal(np.isnan(g), np.isnan(ref))
            assert np.max(np.abs(g - ref), where=~np.isnan(ref), initial=0.0) < TOL
        lk = eng.score_assignments(prm, _dev(truth, eng))
        orc = oracle_score(hb, truth, **kw)
        code = _np(lk["code"])
        assert np.array_equal(code, orc["code"])
        assert np.array_equal(_np(lk["prob_count"]), orc["prob_count"])
        ok = code == 0
        s = _np(lk["score"])
        assert np.array_equal(np.isnan(s), np.isnan(orc["score"]))
        fin = ok & ~np.isnan(s)
        assert np.max(np.abs(s[fin] - orc["score"][fin]), initial=0.0) < TOL
    eng.status()


def _check_solve_outputs(out, hb, probs=None):
    """chosen_code 1 exactly where assign has -1; chosen_score = the oracle's score of the chosen tuple
    under the returned mixtures; margin as defined; service sums against a host sum."""
    orc = oracle_score(hb, out["assign"], mix=out["mixtures"])
    code, score = out["chosen_code"], out["chosen_score"]
    for p in range(hb.n_problems):
        i0, i1 = int(hb.prob_in_off[p]), int(hb.prob_in_off[p + 1])
        t0, t1 = int(hb.prob_tuple_off[p]), int(hb.prob_tuple_off[p + 1])
        n = i1 - i0
        E = (t1 - t0) // n
        a = out["assign"][t0:t1]
        assert np.array_equal(code[i0:i1] == 1, (a.reshape(E, n) < 0).any(axis=0))
        m = host_margin(score[i0:i1], code[i0:i1], a, E, out["topk_score"][i0:i1], out["topk_idx"][K * t0:K * t1],
                        out["topk_cnt"][i0:i1])
        assert np.array_equal(out["margin"][i0:i1], m, equal_nan=True)
        ok = code[i0:i1] == 0
        host = score[i0:i1][ok].sum()
        assert out["service_loglik"][p] == pytest.approx(host, rel=1e-12, abs=1e-9)
        assert np.array_equal(out["service_codes"][p], np.bincount(code[i0:i1], minlength=5))
    assert np.array_equal(code, orc["code"])
    ok = code == 0
    assert np.max(np.abs(score[ok] - orc["score"][ok]), initial=0.0) < TOL
    assert np.array_equal(out["mixture_off"], hb.ep_term_off[hb.prob_ep_off])


def test_solve_likelihood_outputs(solver, golden_batch, batches):
    for hb in (golden_batch[0], batches["hotel"], batches["shapes"], batches["wide"]):
        out = {k: np.array(v) for k, v in solver.solve(hb, want_scores=True, want_likelihood=True,
                                                        want_mixtures=True).items()}
        _check_solve_outputs(out, hb)
        again = solver.solve(hb, want_likelihood=True)
        assert again["service_loglik"].tobytes() == out["service_loglik"].tobytes()


def test_solver_scores_the_truth(solver, golden_batch):
    hb, probs, gauss, mix, truth = golden_batch
    res = solver.score(hb, truth, mix)
    orc = oracle_score(hb, truth, mix=mix)
    assert np.array_equal(res["code"], orc["code"])
    assert np.array_equal(res["service_codes"], orc["prob_count"])
    ok = res["code"] == 0
    assert np.max(np.abs(res["score"][ok] - orc["score"][ok]), initial=0.0) < TOL
    np.testing.assert_allclose(res["service_loglik"], orc["prob_sum"], rtol=1e-12, atol=1e-9)


def test_new_outputs_change_nothing_else(engine, batches):
    """Existing outputs are identical with the new outputs on or off, the default path launches exactly what
    it did, and the likelihood adds two launches (int64 bind)."""
    from traceweaver_b200.predictor import solve_bound
    eng, hb = engine, batches["hotel"]
    eng.bind(hb)
    c0 = eng.launch_count()
    a = solve_bound(eng, seed_select=10)
    c1 = eng.launch_count()
    b = solve_bound(eng, seed_select=10, want_likelihood=True)
    c2 = eng.launch_count()
    c = solve_bound(eng, seed_select=10)
    c3 = eng.launch_count()
    assert c2 - c1 == c1 - c0 + 2
    assert c3 - c2 == c1 - c0
    for k in RESULTS:
        assert _np(a[k]).tobytes() == _np(b[k]).tobytes() == _np(c[k]).tobytes(), k
    assert "likelihood" not in a


def test_chunked_solve_equals_single_group():
    from traceweaver_b200 import synth
    from traceweaver_b200.api import BatchSolver
    from traceweaver_b200.batch import build_batch_from_blocks
    hb = build_batch_from_blocks(synth.hotel_stream(1100, 1000, seed=11))
    assert int(hb.prob_in_off[-1]) > BatchSolver.MIN_CHUNK_IN_SPANS
    one, four = BatchSolver(device=0, chunks=1), BatchSolver(device=0, chunks=4)
    try:
        a = {k: np.array(v) for k, v in one.solve(hb, want_scores=True, want_likelihood=True,
                                                   want_mixtures=True).items()}
        b = four.solve(hb, want_scores=True, want_likelihood=True, want_mixtures=True)
        assert four.last_chunks == 4
        for k in RESULTS + LIKELIHOOD:
            assert a[k].tobytes() == b[k].tobytes(), k
        plain = four.solve(hb, want_scores=True)
        for k in RESULTS:
            assert a[k].tobytes() == plain[k].tobytes(), k
        assert not set(LIKELIHOOD) & set(plain)
    finally:
        one.close()
        four.close()


def test_integral_float_binds_bit_identical(solver, golden_batch):
    from traceweaver_b200.batch import Problem, build_batch
    hb, probs = golden_batch[0], golden_batch[1]
    f = lambda x: np.asarray(x, np.int64).astype(np.float64)
    hf = build_batch([Problem(in_start=f(p.in_start), in_end=f(p.in_end), out_start=[f(x) for x in p.out_start],
                              out_end=[f(x) for x in p.out_end], preds=p.preds, name=p.name) for p in probs])
    assert hf.float_times
    a = {k: np.array(v) for k, v in solver.solve(hb, want_likelihood=True, want_mixtures=True).items()}
    b = solver.solve(hf, want_likelihood=True, want_mixtures=True)
    for k in LIKELIHOOD:
        assert a[k].tobytes() == b[k].tobytes(), k
    truth = golden_batch[4]
    assert solver.score(hb, truth, a["mixtures"])["score"].tobytes() == \
        solver.score(hf, truth, a["mixtures"])["score"].tobytes()


def test_compressed_fixtures_match_the_float_oracle(engine, goldens):
    """Compression divides start times and keeps durations, so the uncompressed truth is mostly infeasible
    there (code 4, as in the float oracle); the engine's own final tuples are scored under its own model."""
    from traceweaver_b200.batch import build_batch
    from traceweaver_b200.predictor import solve_bound
    sel = [g for g in goldens if g.path.split("/")[-1][:-4] in SOLVABLE[3]]
    probs = [compress(g.problem(), 3) for g in sel]
    hb = build_batch(probs)
    truth = np.concatenate([g.z["truth"].astype(np.int32).reshape(-1) for g in sel])
    eng = engine
    eng.bind(hb)
    res = solve_bound(eng, seed_select=10)
    mix = _np(res["params_pass1"].table)
    rank0 = _rank_assign_batch(hb, _np(res["topk_idx"]), _np(res["topk_cnt"]), 0)
    p0 = eng.params_pass0()
    gauss = _np(p0.table)
    n_scored = 0
    for prm, kw in ((res["params_pass1"], dict(mix=mix)), (p0, dict(gauss=gauss))):
        for a in (truth, _np(res["assign"]), rank0):
            lk = eng.score_assignments(prm, _dev(a, eng))
            orc = oracle_score(hb, a, **kw, float_times=True)
            code, s = _np(lk["code"]), _np(lk["score"])
            assert np.array_equal(code, orc["code"])
            assert np.array_equal(np.isnan(s), np.isnan(orc["score"]))
            fin = ~np.isnan(s)
            n_scored += int(fin.sum())
            assert np.max(np.abs(s[fin] - orc["score"][fin]), initial=0.0) < TOL
    assert n_scored > 0
    eng.status()
