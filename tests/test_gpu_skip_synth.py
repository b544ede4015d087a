"""GPU: the skip regime (skipmode.solve -> tw_skip_solve / k_skip, tw_build_dist_samples) on generated
cache-mode services (tests/skip_synth.py) against the oracle (oracle/tw_oracle_skip.py): the whole path
per service including the host mirror's windows, skip counts and services_times table, the scores of
the chosen assignment and of the generator's truth, state carried from service to service through one
SkipState and one Engine, the drop-in predictor's parked two-pass state, engine scratch reuse across
service sizes, and the per-in-span candidate limit."""
import numpy as np
import pytest

import skip_synth as ss
from assess.skip_oracle_assess import assess_service
from oracle import tw_oracle_skip as osk
from test_skip_synth import CASES, IDS
from traceweaver_b200 import _abi, skipmode

pytestmark = pytest.mark.gpu
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


@pytest.fixture(scope="module")
def oracle_runs():
    runs = {}

    def get(name):
        if name not in runs:
            svc = dict(CASES)[name]()
            runs[name] = (svc,) + ss.run_oracle(svc)
        return runs[name]
    return get


def _state(svc):
    st = skipmode.SkipState()
    st.time_windows = list(svc.wins_before)
    st.distribution_values = {k: list(v) for k, v in svc.values_before.items()}
    return st


def _solve(eng, svc, labels=None, state=None, **kw):
    return skipmode.solve(eng, svc.in_start, svc.in_end, svc.out_start, svc.out_end, svc.preds, labels=labels,
                          state=state if state is not None else _state(svc), **kw)


def _check_model(res, ref):
    """The host mirror and k_build_dist: bit-equal to the oracle's model."""
    assert [tuple(w) for w in res["time_windows"]] == [tuple(w) for w in ref["time_windows"]]
    assert list(res["skip_budget"]) == list(ref["skip_budget"])
    assert np.array_equal(np.asarray(res["skip_count"]), np.asarray(ref["skip_count"]))
    assert res["pair_params"].tobytes() == np.asarray(ref["pair_params"], np.float64).tobytes()
    assert res["large_delay"] == ref["large_delay"]


@pytest.mark.parametrize("name", IDS)
def test_engine_equals_oracle(engine, oracle_runs, name):
    svc, ref, _, _ = oracle_runs(name)
    if isinstance(ref, osk.ReferenceUndefined):
        with pytest.raises(_abi.TwError) as ex:
            _solve(engine, svc)
        assert ex.value.code == _abi.TW_ERR_REFERENCE_UNDEFINED, str(ref)
        return
    res = _solve(engine, svc)
    _check_model(res, ref)
    ss.assert_equals_oracle(res, ref)


@pytest.mark.parametrize("name", IDS)
def test_likelihood_equals_oracle_checker(engine, oracle_runs, name):
    """want_likelihood=True: the chosen tuples' scores and codes, and skipmode.score of the generator's
    truth (the cached call as a skip span), against the oracle's scoring code."""
    svc, ref, _, md = oracle_runs(name)
    if isinstance(ref, osk.ReferenceUndefined):
        pytest.skip(f"the reference raises: {ref}")
    res = _solve(engine, svc, want_likelihood=True)
    orc = assess_service(svc.in_start, svc.in_end, svc.out_start, svc.out_end, svc.preds, res["assign"],
                         ref["pair_params"], md["normalized"])
    assert np.array_equal(res["chosen_code"], orc["code"])
    assert np.array_equal(res["service_codes"], orc["service_codes"])
    ok = orc["code"] == 0
    assert np.allclose(res["chosen_score"][ok], orc["score"][ok], rtol=ss.RTOL, atol=0)
    assert np.all(np.isnan(res["chosen_score"][~ok]))
    lk = skipmode.score(engine, svc.in_start, svc.in_end, svc.out_start, svc.out_end, svc.preds, svc.truth, res)
    orc = assess_service(svc.in_start, svc.in_end, svc.out_start, svc.out_end, svc.preds, svc.truth,
                         ref["pair_params"], md["normalized"])
    assert np.array_equal(lk["code"], orc["code"])
    ok = orc["code"] == 0
    assert ok.any()
    assert np.allclose(lk["score"][ok], orc["score"][ok], rtol=ss.RTOL, atol=0)


def _named(svc_labels, dv):
    """Oracle samples are keyed by tuple position: the carried lists of this service's endpoints."""
    E1 = len(svc_labels)
    return {(a, b): list(dv[(svc_labels[a], svc_labels[b])]) for a in range(E1) for b in range(E1)
            if (svc_labels[a], svc_labels[b]) in dv}


def _sequence():
    """Services of different shapes and endpoint names; the second opens its first window at the start of
    the first's, and endpoint names recur, so samples accumulate across services."""
    a = ss.make_service("hotel_search", n=150, load=100.0, seed=51, cached=(1,), rate=0.2)
    b0 = ss.make_service("hotel_frontend", n=150, load=100.0, seed=52, cached=(1,), rate=0.2)
    b = ss.make_service("hotel_frontend", n=150, load=100.0, seed=52, cached=(1,), rate=0.2,
                        shift=int(a.in_start[0]) - int(b0.in_start[0]))
    c = ss.make_service("media_movie_id", n=150, load=60.0, seed=53, quantum=1000, extra=((1, 8),))
    d = ss.make_service("hotel_search", n=150, load=100.0, seed=54, cached=(0,), rate=0.2, quantum=1000)
    e = ss.make_service("dag8", n=100, load=60.0, seed=55, cached=(1,), rate=0.2)
    return [(a, ["search", "geo", "rate"]), (b, ["frontend", "search", "reservation", "profile"]),
            (c, ["movie-id", "rating", "compose"]), (d, ["search", "geo", "rate"]),
            (e, ["gateway"] + [f"svc{k}" for k in range(7)] + ["profile"])]


def test_state_carried_across_services(engine):
    st = skipmode.SkipState()
    wins, dv = [], {}
    seq = _sequence()
    shared = 0
    for svc, labels in seq:
        ref = osk.solve_skip(svc.in_start, svc.in_end, svc.out_start, svc.out_end, svc.preds,
                             time_windows_before=list(wins), values_before=_named(labels, dv))
        assert not isinstance(ref, Exception)
        res = _solve(engine, svc, labels=labels, state=st)
        _check_model(res, ref)
        ss.assert_equals_oracle(res, ref)
        starts = [w[0] for w in ref["time_windows"]]
        shared += len(starts) - len(set(starts))
        wins.extend(osk.new_time_windows([int(x) for x in svc.in_start], [int(x) for x in svc.in_end]))
        for (x, y), v in ref["samples"]:
            dv.setdefault((labels[x], labels[y]), []).append(v)
        assert st.time_windows == wins
        assert {k: list(v) for k, v in st.distribution_values.items()} == dv
    assert shared > 0


def _spans(prefix, svc, labels, G):
    from test_gpu_pipeline import Span
    n = svc.n
    in_spans = [Span(f"{prefix}t{i}", f"{prefix}in{i}", svc.in_start[i], svc.in_end[i] - svc.in_start[i])
                for i in range(n)]
    outs = {}
    for e, ep in enumerate(labels[1:]):
        outs[ep] = [Span(f"{prefix}o{e}", f"{prefix}o{e}.{j}", s, x - s)
                    for j, (s, x) in enumerate(zip(svc.out_start[e], svc.out_end[e]))]
    return {labels[0]: in_spans}, outs


def _graph(labels, preds):
    import networkx as nx
    G = nx.DiGraph()
    G.add_nodes_from(labels[1:])
    for e, pl in enumerate(preds):
        for b in pl:
            G.add_edge(labels[1 + b], labels[1 + e])
    return G


def test_predictor_sequence_replays_parked_state():
    """Two two-pass services, then a cache-mode service, through one TraceWeaverV3: the skip service's
    6-tuple equals the oracle's run with the windows and samples the earlier services leave behind."""
    from traceweaver_b200.predictor import TraceWeaverV3
    first = (ss.make_service("hotel_search", n=150, load=100.0, seed=61), ["search", "geo", "rate"])
    second = (ss.make_service("hotel_frontend", n=150, load=100.0, seed=62),
              ["frontend", "search", "reservation", "profile"])
    skip = (ss.make_service("hotel_frontend", n=150, load=100.0, seed=63, cached=(1,), rate=0.2, quantum=1000),
            ["frontend", "search", "reservation", "profile"])
    pred = TraceWeaverV3({}, {}, device=0)
    wins, dv = [], {}
    try:
        for k, (svc, labels) in enumerate((first, second)):
            G = _graph(labels, svc.preds)
            ins, outs = _spans(f"p{k}", svc, labels, G)
            pred.FindAssignments("MaxScoreBatchSubsetWithSkips", labels[0], ins, outs, False, [], {}, G)
            ii, ie = [int(x) for x in svc.in_start], [int(x) for x in svc.in_end]
            wins.extend(osk.new_time_windows(ii, ie))
            samples, _ = osk.build_distribution_samples(ii, ie, [[int(x) for x in o] for o in svc.out_start],
                                                        [[int(x) for x in o] for o in svc.out_end])
            for (x, y), v in samples:
                dv.setdefault((labels[x], labels[y]), []).append(v)
        svc, labels = skip
        G = _graph(labels, svc.preds)
        ins, outs = _spans("s", svc, labels, G)
        got = pred.FindAssignments("MaxScoreBatchSubsetWithSkips", labels[0], ins, outs, False, [], {}, G)
    finally:
        pred.engine.close()
    ref = osk.solve_skip(svc.in_start, svc.in_end, svc.out_start, svc.out_end, svc.preds,
                         time_windows_before=wins, values_before=_named(labels, dv))
    assert not isinstance(ref, Exception)
    a, topk, not_best, n, cands, unassigned = got
    in_ids = [s.GetId() for s in ins[labels[0]]]
    for e, ep in enumerate(labels[1:]):
        ids = [s.GetId() for s in outs[ep]]

        def name(c):
            return ids[c] if c >= 0 else (("NA", "NA") if c == -1 else ("Skip", "Skip"))
        for i, iid in enumerate(in_ids):
            assert a[ep][iid] == name(int(ref["assign"][e, i])), (ep, i)
            assert topk[ep][iid] == [name(int(c)) for c in ref["topk2_idx"][i, :ref["topk2_cnt"][i], e]], (ep, i)
    assert (not_best, n, unassigned) == (ref["not_best_count"], svc.n, ref["cnt_unassigned"])
    assert cands == {iid: int(ref["n_cand"][i]) for i, iid in enumerate(in_ids) if ref["n_cand"][i]}
    assert (ref["assign"] == -2).any()


def test_engine_reuse_across_sizes_is_bit_identical(engine):
    """Big, small, big on one Engine (scratch only grows; taken bits are cleared per problem) against a
    fresh Engine per service."""
    from traceweaver_b200.engine import Engine
    big = dict(CASES)["media_nginx_cal-n200-L60-s11-q1-c1@0.2-xnone"]()
    small = ss.make_service("hotel_search", n=40, load=100.0, seed=12, cached=(0,), rate=0.2, quantum=1000)
    big2 = dict(CASES)["dag8-n120-L60-s11-q1-c1@0.2-xnone"]()
    reused = [_solve(engine, s) for s in (big, small, big2)]
    for s, r in zip((big, small, big2), reused):
        eng = Engine(0)
        try:
            fresh = _solve(eng, s)
        finally:
            eng.close()
        for k in RESULTS:
            assert np.asarray(r[k]).tobytes() == np.asarray(fresh[k]).tobytes(), (s.name, k)


def test_candidate_limit(engine, oracle_runs):
    """96 candidates of one callee inside one in-span solve like the oracle; 97 are TW_ERR_RANGE_LIMIT and
    no answer comes back; the same engine then solves an ordinary service like the oracle."""
    svc = ss.cand_limit_service(96)
    ref, _, _ = ss.run_oracle(svc)
    res = _solve(engine, svc)
    _check_model(res, ref)
    ss.assert_equals_oracle(res, ref)
    with pytest.raises(_abi.TwError) as ex:
        _solve(engine, ss.cand_limit_service(97))
    assert ex.value.code == _abi.TW_ERR_RANGE_LIMIT
    name = "hotel_frontend-n200-L100-s11-q1-c1@0.2-xnone"
    svc, ref, _, _ = oracle_runs(name)
    res = _solve(engine, svc)
    _check_model(res, ref)
    ss.assert_equals_oracle(res, ref)
