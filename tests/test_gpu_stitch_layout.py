"""GPU vs CPU oracle on batches whose services need different amounts of the stitch kernel's per-warp
shared memory.  The slab is sized per batch, for its largest E and its largest taken bitmap, so these
check the largest packing stride next to the smallest, and a service whose taken bitmap stays in
global memory next to services that fit the batch's shared-memory budget.  Each pass is compared
given the oracle's parameters."""
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


# eight parallel callees (E = 8, the largest the engine takes), no DAG edges
PAR8 = dict(preds=[[]] * 8, eps=[(250 + 40 * e, 0.6, 2500 + 300 * e, 0.6) for e in range(8)],
            tail=(200, 0.7), chain=False)


def _np(t):
    return t.cpu().numpy()


def _check_passes(eng, hb):
    from oracle import tw_oracle
    ob = tw_oracle.OracleBatch(hb)
    eng.bind(hb)
    eng.prepare()
    g_cpu = ob.params_pass0()
    prm = eng.params_from_host(gauss=g_cpu)
    sc = eng.score(prm, want_used=True)
    o_sc = ob.score(gauss=g_cpu)
    eng.status()
    assert np.array_equal(_np(sc["cut"]), o_sc["cut"])
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
    d, c = ob.delays(o_st["assign"])
    mix, _, _ = tw_oracle.gmm_refit(hb.term_sample_off, d, c, seed_select=10)
    prm1 = eng.params_from_host(mix=mix)
    sc1 = eng.score(prm1, want_used=True)
    o_st1 = ob.stitch(o_sc["cut"], mix=mix)
    st1 = eng.stitch(prm1, sc["cut"], undeleted=sc1)
    eng.status()
    assert np.array_equal(_np(st1["assign"]), o_st1["assign"])
    assert np.array_equal(_np(st1["mis_rank"]), o_st1["mis_rank"])


def test_mixed_e1_e8_batch_matches_oracle(engine, monkeypatch):
    """Services of one callee and of eight in one batch: tuples packed at stride 1 and 8 in slabs sized for E = 8."""
    from traceweaver_b200 import synth
    from traceweaver_b200.batch import build_batch_from_blocks
    monkeypatch.setitem(synth.SHAPES, "par8", PAR8)
    hb = build_batch_from_blocks([synth.make_block("single", 4, 300, 300.0, seed=21),
                                  synth.make_block("par8", 3, 200, 150.0, seed=22)])
    E = np.diff(hb.prob_ep_off)
    assert E.min() == 1 and E.max() == 8
    _check_passes(engine, hb)


def test_one_service_over_the_taken_budget_matches_oracle(engine):
    """One service whose taken bitmap (> 256 words) lives in global memory, the others in shared memory."""
    from traceweaver_b200 import synth
    from traceweaver_b200.batch import build_batch_from_blocks
    hb = build_batch_from_blocks([synth.make_block("hotel_frontend", 1, 5000, 100.0, seed=31),
                                  synth.make_block("hotel_frontend", 4, 300, 300.0, seed=32),
                                  synth.make_block("hotel_search", 3, 300, 300.0, seed=33)])
    words = []
    for p in range(hb.n_problems):
        eps = range(int(hb.prob_ep_off[p]), int(hb.prob_ep_off[p + 1]))
        words.append(sum(int(hb.ep_out_off[e + 1] - hb.ep_out_off[e]) // 32 + 3 for e in eps))
    assert max(words) > 256 and sorted(words)[-2] <= 256
    _check_passes(engine, hb)
