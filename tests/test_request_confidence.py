"""Request confidence (traces.request_confidence_host and the per-in-span step of tw_core.cuh stepped on the
CPU), without a GPU.

Hand-built batches check each rule of the definition in traces.py: a single candidate; the chosen tuple at
rank 0, at a later rank and not listed; a duplicate of the chosen tuple in the list; the NA and infeasible
codes; a request with a zero decision; exp underflow; the weakest decision's tie; a detached fragment; a
cycle.  Deep chains from deep_tree_util and random inputs cover the per-request sums.  The CPU build of the
device step (tests/emul/tw_emul_confidence.cpp, through emul_backend) must give the host restatement's arrays
bit for bit on all of them and on the final top-K rows of every golden service.  On the pooled golden services
the share of right in-spans must rise strictly over bins of p."""
import math

import numpy as np
import pytest

import emul_backend
from traceweaver_b200 import _abi

K = _abi.TW_K
KEYS = ("p", "ell", "decisions", "zero", "log_conf", "conf", "weakest", "weakest_p", "est_accuracy", "requests",
        "expected_exact", "q")


def check_same(got, want, keys=KEYS):
    for k in keys:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        assert g.tobytes() == w.astype(g.dtype).tobytes(), k


def everywhere(hb, assign, in_caller, score, code, topk):
    """The host restatement, and the CPU step equal to it bit for bit."""
    from traceweaver_b200.traces import request_confidence_host
    want = request_confidence_host(hb, assign, in_caller, score, code, topk)
    got, rc = emul_backend.request_confidence(hb, assign, want["root"][:int(hb.prob_in_off[-1])], score, code, topk)
    assert rc == 0
    check_same(got, want)
    n_in = int(hb.prob_in_off[-1])
    r = want["root"][:n_in]
    mine = (r >= 0) & (r < n_in)
    assert np.array_equal(want["decisions"], np.bincount(r[mine], minlength=n_in))
    assert ((want["p"] >= 0) & (want["p"] <= 1)).all()
    assert np.array_equal(want["ell"] == np.inf, want["p"] == 0)
    return want


# ------------------------------------------------------------------------------------------------
# hand-built batches: a root service A (one in-span, one call) and a callee service B (one in-span, one call),
# nodes in A = 0, in B = 1, A's call = 2, B's call = 3.  Rows give each in-span's final top-K as (score,
# tuple) pairs; its chosen tuple is index 0 unless `chosen` says otherwise.
# ------------------------------------------------------------------------------------------------
def _pair(links="request"):
    from traceweaver_b200.batch import Problem, build_batch
    t = lambda v: np.array([v], np.int64)
    probs = [Problem(in_start=t(0), in_end=t(100), out_start=[t(10)], out_end=[t(30)], preds=[[]]),
             Problem(in_start=t(12), in_end=t(28), out_start=[t(14)], out_end=[t(20)], preds=[[]])]
    hb = build_batch(probs, validate=False)
    assign, in_caller = {"request": ([0, 0], [-1, 2]), "detached": ([-1, 0], [-1, 2]),
                         "cycle": ([0, 0], [3, 2]), "apart": ([0, 0], [-1, -1])}[links]
    return hb, assign, in_caller


def _inputs(rows, scores, codes):
    n = len(rows)
    ts = np.full((n, K), np.nan)
    ti = np.full((n, K), -1, np.int32)
    cnt = np.zeros(n, np.uint8)
    for i, row in enumerate(rows):
        for r, (s, j) in enumerate(row):
            ts[i, r], ti[i, r] = s, j
        cnt[i] = len(row)
    return np.asarray(scores, np.float64), np.asarray(codes, np.uint8), dict(topk_score=ts, topk_idx=ti.reshape(-1),
                                                                              topk_cnt=cnt)


def _one(row_a, score_a, code_a=0, row_b=((-1.0, 0),), score_b=-1.0, code_b=0, links="request"):
    hb, assign, in_caller = _pair(links)
    score, code, topk = _inputs([row_a, row_b], [score_a, score_b], [code_a, code_b])
    return everywhere(hb, assign, in_caller, score, code, topk)


def _share(sc, others):
    return math.exp(sc) / (math.exp(sc) + sum(math.exp(s) for s in others))


def test_single_candidate_is_certain():
    res = _one([(-3.0, 0)], -3.0)
    assert res["p"][0] == 1.0 and res["ell"][0] == 0.0 and res["q"][0] == 0
    assert res["conf"][0] == 1.0 and res["requests"][0] == 1 and res["decisions"].tolist() == [2, 0]


def test_chosen_at_rank_zero_and_at_a_later_rank():
    res = _one([(-1.0, 0), (-2.0, 1), (-3.0, 2)], -1.0)
    assert res["p"][0] == pytest.approx(_share(-1.0, [-2.0, -3.0]), rel=1e-15)
    assert res["ell"][0] == pytest.approx(-math.log(_share(-1.0, [-2.0, -3.0])), rel=1e-15)
    res = _one([(-1.0, 1), (-2.0, 0), (-3.0, 2)], -2.0)
    assert res["p"][0] == pytest.approx(_share(-2.0, [-1.0, -3.0]), rel=1e-15)


def test_chosen_not_listed_counts_with_its_own_score():
    res = _one([(-1.0, 1), (-2.0, 2)], -5.0)
    assert res["p"][0] == pytest.approx(_share(-5.0, [-1.0, -2.0]), rel=1e-14)


def test_a_duplicate_of_the_chosen_tuple_is_not_an_alternative():
    res = _one([(-1.0, 0), (-2.0, 1), (-1.0, 0)], -1.0)
    assert res["p"][0] == pytest.approx(_share(-1.0, [-2.0]), rel=1e-15)


@pytest.mark.parametrize("code", [_abi.TW_ASSESS_NA, _abi.TW_ASSESS_RANGE, _abi.TW_ASSESS_CONTAIN,
                                  _abi.TW_ASSESS_ORDER])
def test_unscored_choice_is_a_zero_decision(code):
    res = _one([(-1.0, 1)], np.nan, code_a=code, row_b=[(-1.0, 0), (-2.0, 1)], score_b=-1.0)
    assert res["p"][0] == 0.0 and res["ell"][0] == np.inf and res["q"][0] == -1
    assert res["zero"][0] == 1 and res["conf"][0] == 0.0
    assert res["log_conf"][0] == res["q"][1] > 0                       # the other decision still adds up
    assert res["weakest"][0] == 0 and res["weakest_p"][0] == 0.0


def test_exp_underflow_is_a_zero_decision():
    res = _one([(-1.0, 1)], -1000.0)
    assert res["p"][0] == 0.0 and res["ell"][0] == np.inf and res["zero"][0] == 1
    res = _one([(-1.0, 1)], -700.0)                              # tiny but not zero
    assert 0.0 < res["p"][0] < 1e-300 and res["ell"][0] == pytest.approx(699.0, rel=1e-12)


def test_request_sums_and_weakest():
    res = _one([(-1.0, 0), (-2.0, 1)], -1.0, row_b=[(-1.0, 1), (-1.5, 0)], score_b=-1.5)
    pa, pb = _share(-1.0, [-2.0]), _share(-1.5, [-1.0])
    assert res["weakest"][0] == 1 and res["weakest_p"][0] == res["p"][1]
    assert res["log_conf"][0] == res["q"][0] + res["q"][1]
    assert res["conf"][0] == pytest.approx(pa * pb, rel=1e-9)
    assert res["expected_exact"][0] == res["conf"][0]
    assert res["est_accuracy"].tolist() == [res["p"][0], res["p"][1]]
    assert np.isnan(res["conf"][1]) and res["weakest"][1] == -1


def test_weakest_tie_takes_the_smallest_node():
    res = _one([(-1.0, 0), (-2.0, 1)], -1.0, row_b=[(-1.0, 0), (-2.0, 1)], score_b=-1.0)
    assert res["p"][0] == res["p"][1] and res["weakest"][0] == 0


def test_detached_fragment_and_cycle_belong_to_no_request():
    res = _one([(-1.0, 0)], -1.0, links="detached")                # B's caller was taken by no in-span
    assert res["root"][:2].tolist() == [0, 2] and res["decisions"].tolist() == [1, 0]
    assert res["requests"][0] == 1 and np.isnan(res["conf"][1])
    res = _one([(-1.0, 0)], -1.0, links="cycle")
    assert res["root"].tolist() == [-1] * 4 and res["requests"][0] == 0 and res["decisions"].tolist() == [0, 0]
    assert res["expected_exact"][0] == 0.0 and res["p"][0] == 1.0
    res = _one([(-1.0, 0)], -1.0, links="apart")
    assert res["requests"][0] == 2 and res["expected_exact"][0] == res["conf"][0] + res["conf"][1]


def test_malformed_links_and_sizes_raise():
    from traceweaver_b200.traces import request_confidence_host
    hb, _, _ = _pair()
    score, code, topk = _inputs([[(-1.0, 0)], [(-1.0, 0)]], [-1.0, -1.0], [0, 0])
    with pytest.raises(ValueError, match="caller of two"):
        request_confidence_host(hb, [0, 0], [2, 2], score, code, topk)
    with pytest.raises(ValueError, match="topk_idx"):
        request_confidence_host(hb, [0, 0], [-1, 2], score, code, dict(topk, topk_idx=topk["topk_idx"][:3]))
    with pytest.raises(ValueError, match="score and code"):
        request_confidence_host(hb, [0, 0], [-1, 2], score[:1], code, topk)


# ------------------------------------------------------------------------------------------------
# random inputs on any batch: each in-span lists 0..5 tuples, holding its chosen tuple at a random rank or not
# ------------------------------------------------------------------------------------------------
def random_inputs(hb, assign, seed):
    rng = np.random.default_rng(seed)
    n_in = int(hb.prob_in_off[-1])
    assign = np.asarray(assign, np.int32).reshape(-1)
    ts = np.full((n_in, K), np.nan)
    ti = np.full(K * int(hb.prob_tuple_off[-1]), -1, np.int32)
    cnt = rng.integers(0, K + 1, n_in).astype(np.uint8)
    score = np.full(n_in, np.nan)
    code = rng.choice([0, 0, 0, 0, 0, 0, 0, 1, 3], n_in).astype(np.uint8)
    for p in range(hb.n_problems):
        i0, i1 = int(hb.prob_in_off[p]), int(hb.prob_in_off[p + 1])
        n, E, t0 = i1 - i0, int(hb.prob_ep_off[p + 1] - hb.prob_ep_off[p]), int(hb.prob_tuple_off[p])
        chosen = assign[t0:t0 + n * E].reshape(E, n).T
        idx = ti[K * t0:K * (t0 + n * E)].reshape(n, K, E)
        for i in range(n):
            c = int(cnt[i0 + i])
            s = np.sort(rng.normal(-10.0, rng.choice([0.1, 2.0, 50.0]), c))[::-1]
            ts[i0 + i, :c] = s
            idx[i, :c] = rng.integers(0, 4, (c, E))
            at = int(rng.integers(0, c + 1)) if c else 0
            if at < c:
                idx[i, at] = chosen[i]
                score[i0 + i] = s[at]
            else:
                score[i0 + i] = rng.normal(-12.0, 3.0)
            if rng.random() < 0.1 and c > 1:
                idx[i, c - 1] = chosen[i]                             # a duplicate of the chosen tuple
    score[code != 0] = np.nan
    return score, code, dict(topk_score=ts, topk_idx=ti, topk_cnt=cnt)


@pytest.mark.parametrize("depth,spine,seed", [(12, "last", 1), (20, "first", 2), (40, "last", 3)])
def test_deep_chains(depth, spine, seed):
    from deep_tree_util import deep_trees
    t = deep_trees(depth, callees=3, spine=spine, requests=3, random_shape=True, order="shuffled", seed=seed)
    score, code, topk = random_inputs(t["hb"], t["assign"], seed)
    res = everywhere(t["hb"], t["assign"], t["in_caller"], score, code, topk)
    assert sorted(np.flatnonzero(res["root"][:len(res["p"])] == np.arange(len(res["p"])))) == sorted(t["roots"])
    assert res["requests"][0] == 3


def test_trace_directories(tmp_path):
    from test_traces import ALIBABA_DIR, _tree_dir, load_batch
    for layout in ("hotel", "node", "alibaba"):
        directory = ALIBABA_DIR if layout == "alibaba" else _tree_dir(tmp_path, layout, n_req=120)
        _, hb, in_caller, truth, _ = load_batch(directory, layout)
        score, code, topk = random_inputs(hb, truth, 7)
        everywhere(hb, truth, in_caller, score, code, topk)


def test_exp_and_log_are_the_same_on_both_builds():
    from traceweaver_b200.traces import conf_exp, conf_log
    rng = np.random.default_rng(0)
    d = -np.concatenate([np.linspace(0.0, 750.0, 30001), rng.exponential(5.0, 30000), [0.0, 745.5, np.inf]])
    x = np.concatenate([1.0 + rng.random(30000) * 5.0, np.exp(np.linspace(-700, 700, 20001)), [1.0, 6.0]])
    for f, cpu, v in ((conf_exp, emul_backend.conf_exp, d), (conf_log, emul_backend.conf_log, x)):
        got = cpu(v)
        assert got.tobytes() == f(v).tobytes(), f.__name__
    ref = np.exp(d[d > -708])
    assert np.max(np.abs(conf_exp(d[d > -708]) - ref) / ref) < 3e-16
    assert np.max(np.abs(conf_log(x) - np.log(x)) / np.maximum(np.abs(np.log(x)), 1e-300)) < 4e-16
    assert conf_exp(np.array([0.0]))[0] == 1.0 and conf_log(np.array([1.0]))[0] == 0.0


# ------------------------------------------------------------------------------------------------
# the golden services: the reference's last-pass assignment, scored by the oracle, against its final top-K
# ------------------------------------------------------------------------------------------------
BINS = (0.0, 0.5, 0.8, 0.95, 0.99, 0.999, 1.0 + 1e-12)


def golden_choices():
    from golden_util import Golden, golden_files
    from oracle.tw_oracle import OracleBatch
    from traceweaver_b200.batch import build_batch
    from traceweaver_b200.traces import choice_host
    ps, right = [], []
    for f in golden_files():
        g = Golden(f)
        prob = g.problem()
        hb = build_batch([prob])
        a = np.ascontiguousarray(g.z["assign"], np.int32)
        n, E = a.shape[1], a.shape[0]
        top = dict(topk_score=g.z["topk2_score"][1], topk_idx=g.z["topk2_idx"][1].astype(np.int32).reshape(-1),
                   topk_cnt=g.z["topk2_cnt"][1].astype(np.uint8))
        sc = OracleBatch(hb).score_assignments(a.reshape(-1), mix=g.mix_table(prob))
        score = sc["score"].copy()
        listed = (g.z["topk2_idx"][1] == a.T[:, None, :]).all(axis=2) & (np.arange(K) < top["topk_cnt"][:, None])
        at = np.where(listed.any(axis=1), listed.argmax(axis=1), -1)
        score[at >= 0] = top["topk_score"][at >= 0, at[at >= 0]]          # the listed score where it is listed
        p, ell, q = choice_host(hb, a, score, sc["code"], top)
        got, rc = emul_backend.request_confidence(hb, a, np.arange(n, dtype=np.int32), score, sc["code"], top)
        assert rc == 0
        check_same(got, dict(p=p, ell=ell, q=q), keys=("p", "ell", "q"))
        ps.append(p)
        right.append((a == g.z["truth"]).all(axis=0))
    return np.concatenate(ps), np.concatenate(right)


def test_golden_services_rank_right_choices_higher():
    p, right = golden_choices()
    b = np.digitize(p, BINS) - 1
    share = [right[b == k].mean() for k in range(len(BINS) - 1)]
    assert all((b == k).sum() > 100 for k in range(len(BINS) - 1))
    assert all(x < y for x, y in zip(share, share[1:])), share
