"""Scoring a given assignment (tw_score_assignments) on the CPU: the oracle's restatement against the
golden fixtures minted from the reference, crafted tuples for every feasibility code, and the engine's
per-in-span device function (assess_in_span, tw_core.cuh) stepped on the CPU against the oracle."""
import numpy as np
import pytest

from assess_backends import emul_score, oracle_score
from golden_util import Golden, golden_files
from traceweaver_b200 import _abi
from traceweaver_b200.batch import Problem, build_batch

FILES = golden_files()
IDS = [f.split("/")[-1][:-4] for f in FILES]
TOL = 1e-10
K = _abi.TW_K


@pytest.fixture(scope="module", params=FILES, ids=IDS)
def case(request):
    g = Golden(request.param)
    prob = g.problem()
    hb = build_batch([prob])
    return g, prob, hb


def _params(g, prob, pass_id):
    return dict(gauss=g.gauss_table(prob)) if pass_id == 0 else dict(mix=g.mix_table(prob))


def rank_assign(idx, cnt, r):
    """The rank-r tuples of a top-K list (idx [n, K, E]) in tw_pass_out.assign layout; -1 past the count."""
    n, _, E = idx.shape
    a = idx[:, r, :].T.astype(np.int32).copy()
    a[:, cnt <= r] = -1
    return a.reshape(-1)


def host_margin(score, code, assign, E, topk_score, topk_idx, topk_cnt):
    """The margin's definition, restated on the host."""
    n = len(code)
    a = assign.reshape(E, n).T
    idx = topk_idx.reshape(n, K, E)
    m = np.full(n, np.nan)
    for i in range(n):
        if code[i] != 0 or topk_cnt[i] == 0:
            continue
        if np.array_equal(idx[i, 0], a[i]):
            m[i] = topk_score[i, 0] - topk_score[i, 1] if topk_cnt[i] > 1 else np.inf
        else:
            m[i] = score[i] - topk_score[i, 0]
    return m


@pytest.mark.parametrize("pass_id", [0, 1])
@pytest.mark.parametrize("which", ["topk2", "topk"])
def test_oracle_scores_golden_tuples(case, pass_id, which):
    """Every tuple of the golden top-K lists (no-deletion `topk2`, with-deletion `topk`) is feasible and
    scores its listed score."""
    g, prob, hb = case
    idx, cnt, want = (g.z[f"{which}_idx"][pass_id], g.z[f"{which}_cnt"][pass_id], g.z[f"{which}_score"][pass_id])
    for r in range(K):
        live = cnt > r
        if not live.any():
            break
        res = oracle_score(hb, rank_assign(idx, cnt, r), **_params(g, prob, pass_id))
        assert np.all(res["code"][live] == _abi.TW_ASSESS_SCORED)
        assert np.all(res["code"][~live] == _abi.TW_ASSESS_NA)
        got, ref = res["score"][live], want[live, r]
        assert np.array_equal(np.isnan(got), np.isnan(ref))       # NaN where a pass-0 record is NaN
        assert np.max(np.abs(got - ref), where=~np.isnan(ref), initial=0.0) < TOL
        assert np.all(np.isnan(res["score"][~live]))


def test_oracle_scores_the_truth(case):
    g, prob, hb = case
    res = oracle_score(hb, g.z["truth"].astype(np.int32).reshape(-1), mix=g.mix_table(prob))
    code, score = res["code"], res["score"]
    assert np.all(code < _abi.TW_ASSESS_NCODES)
    assert np.all(np.isfinite(score[code == 0])) and np.all(np.isnan(score[code != 0]))
    assert np.array_equal(res["prob_count"][0], np.bincount(code, minlength=_abi.TW_ASSESS_NCODES))
    assert res["prob_sum"][0] == pytest.approx(score[code == 0].sum(), rel=1e-12, abs=1e-12)
    # the reference's own assignment of the last pass is feasible everywhere it assigned
    a = g.z["assign"].astype(np.int32)
    res = oracle_score(hb, a.reshape(-1), mix=g.mix_table(prob))
    assert np.array_equal(res["code"] == _abi.TW_ASSESS_NA, (a < 0).any(axis=0))
    assert np.all(res["code"][(a >= 0).all(axis=0)] == _abi.TW_ASSESS_SCORED)


def test_device_function_equals_oracle(case):
    """assess_in_span stepped on the CPU: codes and counts exact, scores within 1e-10 of the oracle, the
    per-service sum in the kernels' order within 1e-12 of a host sum, margins as defined."""
    g, prob, hb = case
    mix = g.mix_table(prob)
    top = dict(topk_score=g.z["topk2_score"][1], topk_idx=g.z["topk2_idx"][1].astype(np.int32).reshape(-1),
               topk_cnt=g.z["topk2_cnt"][1].astype(np.uint8))
    for a in (g.z["assign"], g.z["truth"], g.z["topk2_idx"][1][:, 1, :].T):
        a = np.ascontiguousarray(a, np.int32).reshape(-1)
        want = oracle_score(hb, a, mix=mix)
        got = emul_score(hb, a, mix=mix, top=top)
        assert np.array_equal(got["code"], want["code"])
        assert np.array_equal(got["prob_count"], want["prob_count"])
        ok = want["code"] == 0
        assert np.all(np.isnan(got["score"][~ok]))
        assert np.max(np.abs(got["score"][ok] - want["score"][ok]), initial=0.0) < TOL
        assert got["prob_sum"][0] == pytest.approx(got["score"][ok].sum(), rel=1e-12, abs=1e-12)
        m = host_margin(got["score"], got["code"], a, prob.E, **top)
        assert np.array_equal(got["margin"], m, equal_nan=True)
    # pass-0 parameters: the record of the in-span's 100-span batch
    gauss = g.gauss_table(prob)
    a = rank_assign(g.z["topk2_idx"][0], g.z["topk2_cnt"][0], 0)
    got = emul_score(hb, a, gauss=gauss)
    live = g.z["topk2_cnt"][0] > 0
    ref = g.z["topk2_score"][0][live, 0]
    assert np.array_equal(np.isnan(got["score"][live]), np.isnan(ref))
    assert np.max(np.abs(got["score"][live] - ref), where=~np.isnan(ref), initial=0.0) < TOL


def crafted():
    """Five in-spans, callee 1 after callee 0 in the DAG, and one tuple per code."""
    n = 5
    in_s = np.arange(n, dtype=np.int64) * 100
    o0s, o0e = in_s + 10, in_s + 30
    o1s, o1e = in_s + 40, in_s + 80
    o0e[4] = 460                      # in-span 4: callee 0 ends after callee 1 starts (440)
    prob = Problem(in_start=in_s, in_end=in_s + 90, out_start=[o0s, o1s], out_end=[o0e, o1e], preds=[[], [0]],
                   name="crafted")
    #                  scored  NA     range  contain order
    assign = np.array([[0, -1, 2, 2, 4],
                       [0, 1, 7, 3, 4]], np.int32)
    return prob, assign, [0, 1, 2, 3, 4]


def test_crafted_codes():
    prob, assign, want = crafted()
    hb = build_batch([prob])
    nterm = int(hb.ep_term_off[-1])
    mix = np.zeros((nterm, _abi.TW_MIX_REC))
    mix[:, 1:4] = (20.0, 5.0, np.log(5.0))             # k = 0: a Gaussian record
    res = oracle_score(hb, assign.reshape(-1), mix=mix)
    assert res["code"].tolist() == want
    assert np.isfinite(res["score"][0]) and np.all(np.isnan(res["score"][1:]))
    assert res["prob_count"][0].tolist() == [1, 1, 1, 1, 1]
    assert res["prob_sum"][0] == res["score"][0]
    got = emul_score(hb, assign.reshape(-1), mix=mix)
    assert got["code"].tolist() == want
    assert abs(got["score"][0] - res["score"][0]) < TOL
    # the lowest code wins: an NA and an out-of-range index in one tuple is NA
    a = assign.copy()
    a[1, 1] = 9
    assert oracle_score(hb, a.reshape(-1), mix=mix)["code"][1] == _abi.TW_ASSESS_NA
    assert emul_score(hb, a.reshape(-1), mix=mix)["code"][1] == _abi.TW_ASSESS_NA
