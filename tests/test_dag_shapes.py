"""The stepped device code (tests/emul) against the oracle on two-pass services of five to eight callees
and up to 28 score terms, and on callees with several primary in-edges listed out of ascending order
(their edge terms are summed in in_edges order, not in topological order).  The shapes are
tests/skip_synth.DAG_SHAPES; each runs at microsecond clocks and at millisecond clocks, where equal
timestamps, zero-length gaps and exact score ties are common.  Scores must be bit-equal: a different
summation order of a callee's terms changes the last bits, nothing else here would see it.  CPU only."""
from functools import lru_cache, partial

import numpy as np
import pytest

import skip_synth
from emul_backend import EmulBatch
from oracle import tw_oracle
from traceweaver_b200.batch import build_batch

# clock -> (timestamp grid in us, mean inter-arrival in us): loads at which the oracle's exact window
# search finishes on every shape
CLOCKS = {"us": (1, 12_000.0), "ms": (1000, 20_000.0)}
N_IN = 260
CASES = [f"{s}-{c}" for s in skip_synth.DAG_SHAPES for c in CLOCKS]

BACKENDS = {"emul": EmulBatch, "emul-lazy": partial(EmulBatch, table_cap=0),
            "emul-combos": partial(EmulBatch, light_combos=0)}


def service(case):
    """(Problem, truth [E, n]) of a case id `<shape>-<clock>`."""
    shape, clock = case.rsplit("-", 1)
    q, ia = CLOCKS[clock]
    return skip_synth.dag_problem(shape, N_IN, ia, seed=4, quantum=q)


@lru_cache(maxsize=None)
def oracle_run(case):
    """Every pass of the oracle on one case: pass-0 Gaussians, score and stitch, the refit on the
    stitch's delays, pass-1 score and stitch under those mixtures."""
    prob, truth = service(case)
    hb = build_batch([prob])
    ob = tw_oracle.OracleBatch(hb)
    g = ob.params_pass0()
    sc = ob.score(gauss=g)
    st = ob.stitch(sc["cut"], gauss=g)
    d, c = ob.delays(st["assign"])
    mix, _, _ = tw_oracle.gmm_refit(hb.term_sample_off, d, c, seed_select=10)
    return dict(prob=prob, truth=truth, hb=hb, gauss=g, sc=sc, st=st, delays=(d, c), mix=mix,
                sc1=ob.score(mix=mix), st1=ob.stitch(sc["cut"], mix=mix))


def _bits_equal(a, b):
    return np.asarray(a, np.float64).tobytes() == np.asarray(b, np.float64).tobytes()


def assert_score_equal(got, ref, what):
    for k in ("cut", "n_feasible", "topk_cnt", "topk_idx"):
        assert np.array_equal(got[k], ref[k]), f"{what}: {k}"
    assert _bits_equal(got["topk_score"], ref["topk_score"]), f"{what}: topk_score"


def assert_stitch_equal(got, ref, what):
    for k in ("assign", "mis_rank", "n_cand", "topk_cnt", "topk_idx"):
        assert np.array_equal(got[k], ref[k]), f"{what}: {k}"
    assert _bits_equal(got["topk_score"], ref["topk_score"]), f"{what}: topk_score"
    assert np.array_equal(got["counters"][:, :2], ref["counters"][:, :2]), f"{what}: counters"


@pytest.mark.parametrize("case", CASES)
def test_generated_service(case):
    """The builder's output is a valid service with the shape's term count, and its truth is a feasible
    tuple of every in-span (code 0) under both passes' parameters."""
    r = oracle_run(case)
    prob = r["prob"]
    prob.validate()
    assert prob.in_accelerated_regime()
    assert len(prob.terms()) == skip_synth.DAG_SHAPES[case.rsplit("-", 1)[0]][1]
    ob = tw_oracle.OracleBatch(r["hb"])
    for kw in (dict(gauss=r["gauss"]), dict(mix=r["mix"])):
        res = ob.score_assignments(r["truth"].reshape(-1), **kw)
        assert np.all(res["code"] == 0), kw.keys()
        assert np.all(np.isfinite(res["score"]))
    if case.endswith("-ms"):   # the millisecond clocks really produce tied scores
        s = r["sc"]["topk_score"]
        assert int((s[:, 1:] == s[:, :-1]).sum()) > 0


@pytest.mark.parametrize("backend", list(BACKENDS))
@pytest.mark.parametrize("case", CASES)
def test_stepped_device_code_equals_oracle(case, backend):
    r = oracle_run(case)
    eb = BACKENDS[backend](r["hb"])
    assert_score_equal(eb.score(gauss=r["gauss"]), r["sc"], "pass-0 score")
    assert_stitch_equal(eb.stitch(r["sc"]["cut"], gauss=r["gauss"]), r["st"], "pass-0 stitch")
    assert_score_equal(eb.score(mix=r["mix"]), r["sc1"], "pass-1 score")
    assert_stitch_equal(eb.stitch(r["sc"]["cut"], mix=r["mix"]), r["st1"], "pass-1 stitch")
    truth = r["truth"].reshape(-1)
    ob = tw_oracle.OracleBatch(r["hb"])
    for kw in (dict(gauss=r["gauss"]), dict(mix=r["mix"])):
        got, ref = eb.score_assignments(truth, **kw), ob.score_assignments(truth, **kw)
        assert np.array_equal(got["code"], ref["code"])
        assert np.array_equal(got["prob_count"], ref["prob_count"])
        assert _bits_equal(got["score"], ref["score"])
