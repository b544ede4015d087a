"""Scoring a given assignment of a cache-mode service (tw_skip_score_assignments) on the CPU: the skip
oracle's scoring code against the golden fixtures minted from the reference with --cache_rate, the
engine's per-in-span device function (skip_assess_in_span, tw_skip_core.cuh) stepped on the CPU against
the goldens and the oracle, and crafted tuples for every feasibility code."""
import numpy as np
import pytest

from assess.skip_emul_assess import emul_skip_score
from assess.skip_oracle_assess import assess, assess_service, scorer
from golden_util import Golden
from oracle import tw_oracle_skip as osk
from test_skip_mode import FILES, IDS
from traceweaver_b200 import _abi

K = _abi.TW_K
ORACLE_RTOL = 1e-15     # test_skip_mode: the oracle's NumPy arithmetic against the reference
DEVICE_RTOL = 1e-12     # test_skip_mode: device exp() against NumPy's


def model(prob, wins_before):
    """The skip regime's model of a service as the oracle builds it: windows, skip counts, budgets, the
    services_times table of BuildDistributions and whether scores are normalised."""
    sorted_start = [sorted(int(x) for x in o) for o in prob.out_start]
    order = [sorted(range(len(o)), key=lambda j, o=o: float(o[j])) for o in prob.out_start]
    sorted_end = [[int(o[j]) for j in od] for o, od in zip(prob.out_end, order)]
    wins, budgets, counts = osk.tally_skip_spans([int(x) for x in prob.in_start], [int(x) for x in prob.in_end],
                                                 sorted_start, list(wins_before))
    samples, _ = osk.build_distribution_samples(prob.in_start, prob.in_end, sorted_start, sorted_end)
    return dict(wins=wins, counts=counts, budgets=budgets, tab=osk.pair_params(samples, prob.E),
                normalized=any(b > 0 for b in budgets))


@pytest.fixture(scope="module", params=FILES, ids=IDS)
def case(request):
    g = Golden(request.param)
    prob = g.problem()
    return g, prob, model(prob, [tuple(w) for w in g.meta["time_windows_before"]])


def rank_tuples(idx, cnt, r):
    """The rank-r tuples of a top-K list (idx [n, K, E]) as an assignment [E, n]; -1 past the count."""
    a = idx[:, r, :].T.astype(np.int32).copy()
    a[:, cnt <= r] = -1
    return a


def truth_with_skips(g, prob):
    """The golden truth with -1 read as the cached call (a skip span) on callees whose list is shorter."""
    t = g.z["truth"].astype(np.int32).copy()
    for e, o in enumerate(prob.out_start):
        if len(o) < prob.n_in:
            t[e][t[e] == -1] = -2
    return t


def host_margin(score, code, assign, top2_score, top2_idx, top2_cnt):
    """The margin's definition against a top2 list, restated on the host (any two skips at a position equal)."""
    m = np.full(len(code), np.nan)
    for i in range(len(code)):
        if code[i] != 0 or top2_cnt[i] == 0:
            continue
        c, t = assign[:, i], top2_idx[i, 0]
        if all(x == y or (x <= -2 and y <= -2) for x, y in zip(c, t)):
            m[i] = top2_score[i, 0] - top2_score[i, 1] if top2_cnt[i] > 1 else np.inf
        else:
            m[i] = score[i] - top2_score[i, 0]
    return m


def _emul(prob, md, assign, top2=None):
    return emul_skip_score(prob.in_start, prob.in_end, prob.out_start, prob.out_end, prob.preds, assign, md["wins"],
                           md["counts"], md["tab"], md["budgets"], top2=top2)


def _oracle(prob, md, assign):
    return assess_service(prob.in_start, prob.in_end, prob.out_start, prob.out_end, prob.preds, assign, md["tab"],
                          md["normalized"])


def _golden_top2(g):
    return dict(top2_score=g.z["topk2_score"][0], top2_idx=g.z["topk2_idx"][0], top2_cnt=g.z["topk2_cnt"][0])


@pytest.mark.parametrize("which", ["topk2", "topk"])
def test_oracle_scores_golden_tuples(case, which):
    """Every tuple of the golden top-K lists (no-deletion `topk2`, with-deletion `topk`) is scored by the
    oracle's own scoring code to its golden score."""
    g, prob, md = case
    idx, cnt, want = g.z[f"{which}_idx"][0], g.z[f"{which}_cnt"][0], g.z[f"{which}_score"][0]
    for r in range(K):
        live = cnt > r
        if not live.any():
            break
        res = _oracle(prob, md, rank_tuples(idx, cnt, r))
        assert np.all(res["code"][live] == 0) and np.all(res["code"][~live] == 1)
        assert np.allclose(res["score"][live], want[live, r], rtol=ORACLE_RTOL, atol=0)


@pytest.mark.parametrize("which", ["topk2", "topk"])
def test_device_function_scores_golden_tuples(case, which):
    """skip_assess_in_span stepped on the CPU: code 0 and the golden score of every listed tuple; the margin
    against the golden top2 list as defined; the service sum in the kernels' order against a host sum."""
    g, prob, md = case
    idx, cnt, want = g.z[f"{which}_idx"][0], g.z[f"{which}_cnt"][0], g.z[f"{which}_score"][0]
    top2 = _golden_top2(g)
    for r in range(K):
        live = cnt > r
        if not live.any():
            break
        a = rank_tuples(idx, cnt, r)
        res = _emul(prob, md, a, top2)
        assert np.all(res["code"][live] == 0) and np.all(res["code"][~live] == 1)
        assert np.allclose(res["score"][live], want[live, r], rtol=DEVICE_RTOL, atol=0)
        assert np.all(np.isnan(res["score"][~live]))
        assert np.array_equal(res["margin"], host_margin(res["score"], res["code"], a, **top2), equal_nan=True)
        assert res["service_score"] == pytest.approx(res["score"][live].sum(), rel=1e-12)
        assert res["service_codes"].tolist() == np.bincount(res["code"], minlength=6).tolist()
    if which == "topk2":     # rank 0 of the list it is measured against: the gap to rank 1
        res = _emul(prob, md, rank_tuples(idx, cnt, 0), top2)
        two = cnt > 1
        assert np.array_equal(res["margin"][two], want[two, 0] - want[two, 1])


def test_truth_stepped_equals_oracle(case):
    """The golden truth (the cached call as a skip span): the stepped device function equals the oracle
    checker code for code, scores within the device tolerance."""
    g, prob, md = case
    t = truth_with_skips(g, prob)
    want = _oracle(prob, md, t)
    got = _emul(prob, md, t)
    assert np.array_equal(got["code"], want["code"])
    assert np.array_equal(got["service_codes"], want["service_codes"])
    ok = want["code"] == 0
    assert ok.sum() > 0.5 * prob.n_in
    assert np.allclose(got["score"][ok], want["score"][ok], rtol=DEVICE_RTOL, atol=0)
    assert np.all(np.isnan(got["score"][~ok]))
    # the reference's own final assignment: unassigned exactly where it has ("NA", "NA")
    a = g.z["assign"].astype(np.int32)
    got = _emul(prob, md, a)
    assert np.array_equal(got["code"] == 1, (a == -1).any(axis=0))
    assert np.all(got["code"][(a != -1).all(axis=0)] == 0)


def crafted():
    """Eight in-spans of a chain 0 -> 1 -> 2 (callee 2 also after 0 is implied only through 1), and one
    tuple per code; in-span 7 skips callee 0, whose pair (incoming, callee 1) is then scored."""
    from traceweaver_b200.batch import Problem
    n = 8
    in_s = np.arange(n, dtype=np.int64) * 100
    outs = [(in_s + 10, in_s + 20), (in_s + 30, in_s + 40), (in_s + 50, in_s + 60)]
    outs[0][1][4] = 435                 # in-span 4: callee 0 ends after callee 1 starts (430)
    prob = Problem(in_start=in_s, in_end=in_s + 90, out_start=[o[0] for o in outs], out_end=[o[1] for o in outs],
                   preds=[[], [0], [1]], name="crafted")
    #                  scored NA  range contain order all-skip chain skip-0
    assign = np.array([[0, -1, 2, 4, 4, -2, -2, -2],
                       [0, 1, 99, 3, 4, -2, -2, 7],
                       [0, 1, 2, 3, 4, -2, 6, 7]], np.int32)
    tab = np.zeros((4, 4, 2))
    tab[..., 0], tab[..., 1] = 10.0, 5.0
    md = dict(wins=[(0, 790, 30)], counts=[[0], [0], [0]], budgets=[1, 0, 0], tab=tab, normalized=True)
    return prob, assign, md, [0, 1, 2, 3, 4, 5, 5, 0]


def test_crafted_codes():
    prob, assign, md, want = crafted()
    for res in (_oracle(prob, md, assign), _emul(prob, md, assign)):
        assert res["code"].tolist() == want
        ok = np.array(want) == 0
        assert np.all(np.isfinite(res["score"][ok])) and np.all(np.isnan(res["score"][~ok]))
        assert res["service_codes"].tolist() == [2, 1, 1, 1, 1, 2]
    a, b = _oracle(prob, md, assign), _emul(prob, md, assign)
    ok = np.array(want) == 0
    assert np.allclose(a["score"][ok], b["score"][ok], rtol=DEVICE_RTOL, atol=0)
    # a missing services_times key on the pair the skip makes the tuple read: the reference raises
    md2 = dict(md, tab=md["tab"].copy())
    md2["tab"][0, 2] = np.nan
    assert _oracle(prob, md2, assign)["code"][7] == 5 and _emul(prob, md2, assign)["code"][7] == 5
    # the lowest code wins: an NA and an out-of-range index in one tuple is NA; a skip's identity is ignored
    a2 = assign.copy()
    a2[1, 1] = 99
    a2[0, 7] = -9
    for res in (_oracle(prob, md, a2), _emul(prob, md, a2)):
        assert res["code"][1] == 1 and res["code"][7] == 0
    assert _emul(prob, md, a2)["score"][7] == b["score"][7]
    # unnormalised (no positive budget): a sum of log densities
    md3 = dict(md, budgets=[0, 0, 0], normalized=False)
    x, y = _oracle(prob, md3, assign), _emul(prob, md3, assign)
    assert np.allclose(x["score"][ok], y["score"][ok], rtol=DEVICE_RTOL, atol=0)
    assert np.all(x["score"][ok] < 0) and np.all(a["score"][ok] > 0)


def test_single_assess_matches_service():
    prob, assign, md, want = crafted()
    ins = [int(x) for x in prob.in_start]
    ine = [int(x) for x in prob.in_end]
    os_ = [[int(x) for x in o] for o in prob.out_start]
    oe_ = [[int(x) for x in o] for o in prob.out_end]
    fn = scorer(ins, ine, os_, oe_, prob.preds, md["tab"], True)
    codes = [assess(fn, i, list(assign[:, i]), ins, ine, os_, oe_, prob.preds)[0] for i in range(prob.n_in)]
    assert codes == want
