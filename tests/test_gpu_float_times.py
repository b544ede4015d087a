"""GPU: float64 microsecond timestamps (time-compressed services, executor.py --compress_factor > 1)
through tw_engine_bind_f64 and the two-pass path, against the int64 path on integral inputs and against
the float64 build of the oracle (tests/oracle_f64.py) on fractional ones."""
import numpy as np
import pytest

from float_times_util import SOLVABLE, compress
from golden_util import Golden, golden_files

pytestmark = pytest.mark.gpu
FILES = golden_files(gpu=True)
FACTORS = (3, 200, 15000)
RESULTS = ("assign", "topk_idx", "topk_cnt", "n_cand", "counters", "mis_rank", "topk_score")


def _np(t):
    return t.cpu().numpy()


def _float_copy(prob):
    from traceweaver_b200.batch import Problem
    f = lambda a: np.asarray(a, np.int64).astype(np.float64)
    return Problem(in_start=f(prob.in_start), in_end=f(prob.in_end), out_start=[f(a) for a in prob.out_start],
                   out_end=[f(a) for a in prob.out_end], preds=prob.preds, name=prob.name)


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


def test_integral_float_inputs_are_bit_identical(solver, goldens):
    from traceweaver_b200.batch import build_batch
    probs = [g.problem() for g in goldens]
    hi, hf = build_batch(probs), build_batch([_float_copy(p) for p in probs])
    assert hf.float_times
    a = {k: np.array(v) for k, v in solver.solve(hi, want_scores=True).items()}
    b = solver.solve(hf, want_scores=True)
    for k in RESULTS:
        assert a[k].tobytes() == b[k].tobytes(), k


@pytest.mark.parametrize("cf", FACTORS)
def test_fractional_inputs_match_the_float_oracle(engine, goldens, cf):
    import oracle_f64
    from traceweaver_b200.batch import build_batch
    probs = [compress(g.problem(), cf) for g in _solvable(goldens, cf)]
    hb = build_batch(probs)
    eng = engine
    eng.bind(hb)
    eng.prepare()
    ob = oracle_f64.OracleBatch(hb)
    # pass-0 parameters: the exact batch sums, rounded once; tstd on the real batch means
    g0 = ob.params_pass0()
    p0 = _np(eng.params_pass0().table)
    eng.status()
    assert np.array_equal(p0[:, 0], g0[:, 0], equal_nan=True)
    np.testing.assert_allclose(p0[:, 1], g0[:, 1], rtol=1e-12)
    np.testing.assert_allclose(p0[:, 2], g0[:, 2], rtol=0, atol=1e-12)
    # windows, candidate counts and the undeleted top-K with the same parameters
    prm0 = eng.params_from_host(gauss=g0)
    sc = eng.score(prm0, want_used=True)
    osc = ob.score(gauss=g0)
    for k in ("cut", "n_feasible", "topk_idx", "topk_cnt"):
        assert np.array_equal(_np(sc[k]), osc[k]), k
    np.testing.assert_allclose(_np(sc["topk_score"]), osc["topk_score"], rtol=1e-12, atol=1e-5, equal_nan=True)
    # iteration 0
    r0 = eng.stitch(prm0, sc["cut"], undeleted=sc, want_topk=True)
    or0 = ob.stitch(osc["cut"], gauss=g0)
    for k in ("assign", "mis_rank", "n_cand", "topk_idx", "topk_cnt"):
        assert np.array_equal(_np(r0[k]), or0[k]), k
    assert np.array_equal(_np(r0["counters"])[:, :2], or0["counters"][:, :2])
    np.testing.assert_allclose(_np(r0["topk_score"]), or0["topk_score"], rtol=1e-12, atol=1e-5, equal_nan=True)
    # delays in real microseconds, identical to the double subtractions
    d, c = eng.delays(r0["assign"])
    od, oc = ob.delays(or0["assign"])
    d, c = _np(d), _np(c)
    assert np.array_equal(c, oc)
    for o, n in zip(hb.term_sample_off[:-1], oc):
        assert d[o:o + n].tobytes() == od[o:o + n].tobytes()
    # refit on those delays: the oracle's driver uses the same stream convention (seed per service, term order)
    prm1, nsel = eng.gmm_refit(torch_tensor(d, eng), torch_tensor(c, eng), seed_select=10, want_selected=True)
    ofa = oracle_f64.find_assignments(hb, 10)
    mix, omix = _np(prm1.table), ofa["mix"]
    nsel = _np(nsel)
    term_prob = np.repeat(np.arange(hb.n_problems), np.diff(hb.ep_term_off[hb.prob_ep_off]))
    node = np.array(["node" in p.name for p in probs])[term_prob]
    same_k = mix[:, 0] == omix[:, 0]
    assert np.all(same_k | node)               # nodejs: ill-conditioned BIC arg-mins (tests/test_gpu_pipeline.py)
    for t in np.flatnonzero(same_k):
        k = int(mix[t, 0])
        w = 3 if k == 0 else k
        np.testing.assert_allclose(mix[t, 1:1 + w], omix[t, 1:1 + w], rtol=1e-7, atol=1e-7)
        if k:
            np.testing.assert_allclose(mix[t, 6:6 + k], omix[t, 6:6 + k], rtol=1e-7, atol=1e-7)
            np.testing.assert_allclose(mix[t, 11:21], omix[t, 11:21], rtol=0, atol=1e-7)
    # iteration 1 with the oracle's mixtures
    prm1 = eng.params_from_host(mix=omix)
    top = eng.score(prm1, out=dict(used_lo=sc["used_lo"], used_bits=sc["used_bits"], used_wide=sc["used_wide"],
                                   cut=sc["cut"]), keep_windows=True)
    otop = ob.score(mix=omix)
    for k in ("topk_idx", "topk_cnt", "n_feasible"):
        assert np.array_equal(_np(top[k]), otop[k]), k
    np.testing.assert_allclose(_np(top["topk_score"]), otop["topk_score"], rtol=1e-12, atol=1e-5, equal_nan=True)
    r1 = eng.stitch(prm1, sc["cut"], undeleted=top)
    or1 = ob.stitch(osc["cut"], mix=omix, want_topk=False)
    eng.status()
    for k in ("assign", "mis_rank", "n_cand"):
        assert np.array_equal(_np(r1[k]), or1[k]), k
    assert np.array_equal(_np(r1["counters"])[:, :2], or1["counters"][:, :2])


def _solvable(goldens, cf):
    return [g for g in goldens if g.path.split("/")[-1][:-4] in SOLVABLE[cf]]


def torch_tensor(a, eng):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)


def test_mixed_batch_keeps_integral_services_bit_identical(solver, goldens):
    from traceweaver_b200.batch import build_batch
    probs = [g.problem() for g in _solvable(goldens, 15000)[:12]]
    mixed = []
    for k, p in enumerate(probs):
        mixed.append(_float_copy(p))
        mixed.append(compress(p, 15000 if k % 2 else 3))
    hm = build_batch(mixed)
    got = {k: np.array(v) for k, v in solver.solve(hm, want_scores=True).items()}
    hi = build_batch(probs)
    want = solver.solve(hi, want_scores=True)
    for k, p in enumerate(probs):
        q = 2 * k                                   # the integral copy of service k in the mixed batch
        for name, w in (("assign", 1), ("topk_idx", 5), ("n_cand", 1), ("mis_rank", 1), ("topk_cnt", 1),
                        ("topk_score", 5)):
            off = "prob_tuple_off" if name in ("assign", "topk_idx") else "prob_in_off"
            om, oi = getattr(hm, off), getattr(hi, off)
            a = got[name].reshape(-1)[w * int(om[q]):w * int(om[q + 1])]
            b = want[name].reshape(-1)[w * int(oi[k]):w * int(oi[k + 1])]
            assert a.tobytes() == b.tobytes(), (name, p.name)
        assert got["counters"][q].tobytes() == want["counters"][k].tobytes()


def _float_stream(S=48, n=300, cf=3.0):
    from traceweaver_b200 import synth
    from traceweaver_b200.batch import ServiceBlock
    out = []
    for b in synth.hotel_stream(S, n, seed=11):
        f = lambda s: s.astype(np.float64) / cf
        out.append(ServiceBlock(in_start=f(b.in_start), in_end=f(b.in_start) + (b.in_end - b.in_start),
                                out_start=[f(s) for s in b.out_start],
                                out_end=[f(s) + (e - s) for s, e in zip(b.out_start, b.out_end)],
                                preds=b.preds, truth=b.truth, name=b.name))
    return out


def test_chunking_gives_identical_results():
    from traceweaver_b200.api import BatchSolver
    from traceweaver_b200.batch import build_batch_from_blocks
    hb = build_batch_from_blocks(_float_stream())
    assert hb.float_times
    one = BatchSolver(device=0, chunks=1)
    four = BatchSolver(device=0, chunks=4)
    four.MIN_CHUNK_IN_SPANS = 0
    a = {k: np.array(v) for k, v in one.solve(hb, want_scores=True).items()}
    b = four.solve(hb, want_scores=True)
    assert four.last_chunks == 4
    for k in RESULTS:
        assert a[k].tobytes() == b[k].tobytes(), k
    one.close()
    four.close()


class Span:
    def __init__(self, trace_id, sid, start_mus, duration_mus):
        self.trace_id, self.sid, self.start_mus, self.duration_mus = trace_id, sid, start_mus, int(duration_mus)

    def GetId(self):
        return (self.trace_id, self.sid)


def _call_args(g, cf):
    """executor.py's FindAssignments arguments after --compress_factor cf (start_mus / cf, floats)."""
    import networkx as nx
    z, m = g.z, g.meta
    in_spans = [Span(t, s, int(a) / cf, d) for t, s, a, d in zip(z["in_trace"], z["in_sid"], z["in_start"], z["in_dur"])]
    out_parts = {}
    for k, ep in enumerate(m["out_eps_given"]):
        out_parts[ep] = [Span(t, s, int(a) / cf, d) for t, s, a, d in
                         zip(z[f"out{k}_trace"], z[f"out{k}_sid"], z[f"out{k}_start"], z[f"out{k}_dur"])]
    G = nx.DiGraph()
    G.add_nodes_from(m["graph_nodes"])
    G.add_edges_from([tuple(e) for e in m["graph_edges"]])
    truth = {}
    for e, ep in enumerate(g.topo):
        truth[ep] = {in_spans[i].GetId(): out_parts[ep][j].GetId() for i, j in enumerate(z["truth"][e]) if j >= 0}
    return {m["in_ep"]: in_spans}, out_parts, truth, G


def test_predictor_solves_fractional_start_times(goldens):
    import oracle_f64
    from traceweaver_b200.batch import build_batch
    from traceweaver_b200.predictor import TraceWeaverV3
    pred = TraceWeaverV3({}, {}, device=0, seed_select=10)
    g = next(g for g in _solvable(goldens, 200) if "node" not in g.name)
    in_parts, out_parts, truth, G = _call_args(g, 200)
    res = pred.FindAssignments("MaxScoreBatchSubsetWithSkips", g.meta["process"], in_parts, out_parts, False, [], truth, G)
    all_assign, all_topk, not_best, num_spans, per_span_cand, cnt_un = res
    last = pred.last
    # the float oracle on the same arrays: iteration 0 outright, iteration 1 given the engine's refit
    prob = compress(g.problem(), 200)
    hb = build_batch([prob])
    ob = oracle_f64.OracleBatch(hb)
    g0 = ob.params_pass0()
    osc = ob.score(gauss=g0)
    or0 = ob.stitch(osc["cut"], gauss=g0, want_topk=False)
    assert np.array_equal(_np(last["assign_pass0"]), or0["assign"])
    mix = _np(last["params_pass1"].table)
    otop = ob.score(mix=mix)
    or1 = ob.stitch(osc["cut"], mix=mix, want_topk=False)
    n, E = prob.n_in, prob.E
    in_ids = [s.GetId() for s in sorted(list(in_parts.values())[0], key=lambda x: float(x.start_mus))]
    assert num_spans == n
    assert not_best == or1["counters"][0, 0] and cnt_un == or1["counters"][0, 1]
    oa, ti = or1["assign"].reshape(E, n), otop["topk_idx"].reshape(n, 5, E)
    for e, ep in enumerate(g.topo):
        ids = [s.GetId() for s in sorted(out_parts[ep], key=lambda x: float(x.start_mus))]
        assert all_assign[ep] == {in_ids[i]: (ids[j] if j >= 0 else ("NA", "NA")) for i, j in enumerate(oa[e])}
        assert all_topk[ep] == {in_ids[i]: [ids[ti[i, r, e]] for r in range(otop["topk_cnt"][i])] for i in range(n)}
    assert [per_span_cand.get(i, 0) for i in in_ids] == (or0["n_cand"] + or1["n_cand"]).tolist()
    # out of scope: fractional times with skip budgets, and a skip service after parked fractional state
    ep = list(out_parts)[0]
    short = dict(out_parts)
    short[ep] = out_parts[ep][:-1]
    with pytest.raises(NotImplementedError):
        pred.FindAssignments("MaxScoreBatchSubsetWithSkips", g.meta["process"], in_parts, short, False, [], truth, G)
    ip, op, tr, G2 = _call_args(g, 1)
    op[ep] = op[ep][:-1]
    with pytest.raises(NotImplementedError):
        pred.FindAssignments("MaxScoreBatchSubsetWithSkips", g.meta["process"], ip, op, False, [], tr, G2)


@pytest.mark.parametrize("bad,code", [(float("nan"), "TW_ERR_INVALID"), (float("inf"), "TW_ERR_INVALID"),
                                      (2.0 ** 56, "TW_ERR_RANGE_LIMIT")])
def test_rejections_name_the_problem(engine, goldens, bad, code):
    from traceweaver_b200 import _abi
    from traceweaver_b200.batch import build_batch
    probs = [compress(g.problem(), 200) for g in goldens[:3]]
    p = probs[1]
    p.out_end[0] = p.out_end[0].copy()
    p.out_end[0][-1] = bad
    hb = build_batch(probs, validate=False)
    with pytest.raises(_abi.TwError) as ex:
        engine.bind(hb)
    assert _abi.STATUS[ex.value.code] == code
    assert "problem 1" in str(ex.value)
    engine.bind(build_batch(probs[:1]))        # the engine stays usable
    engine.prepare()
    engine.params_pass0()
    engine.status()
