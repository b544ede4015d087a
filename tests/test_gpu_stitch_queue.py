"""The stitch kernel's unit queue: a persistent grid whose warps take units (stretches of a service between
strong cuts, or whole services when no candidate maps are given) until the list is empty.  Checked on a
batch of more than 4096 services against the CPU oracle, and on a one-block grid, where two warps take
every unit of every service one after the other, against the default grid."""
import ctypes as C

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
    eng.lib.tw_debug_stitch_grid.argtypes = [C.c_void_p, C.c_int]
    yield eng
    eng.close()


def _np(t):
    return t.cpu().numpy()


KEYS = ("assign", "mis_rank", "n_cand", "counters")


def _pass0(eng, hb):
    """Bind, score under the oracle's pass-0 parameters; returns (params, undeleted lists, oracle stitch)."""
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
    return prm, sc, ob.stitch(o_sc["cut"], gauss=g_cpu)


def _stitch(eng, prm, sc, und):
    st = eng.stitch(prm, sc["cut"], undeleted=und)
    eng.status()
    return {k: _np(st[k]) for k in KEYS}


def _equal_oracle(st, o_st):
    assert np.array_equal(st["assign"], o_st["assign"])
    assert np.array_equal(st["mis_rank"], o_st["mis_rank"])
    assert np.array_equal(st["n_cand"], o_st["n_cand"])
    assert np.array_equal(st["counters"][:, :2], o_st["counters"][:, :2])


def test_batch_over_4096_services_matches_oracle(engine):
    """4,300 services, three of them long enough to split into several units."""
    from traceweaver_b200 import synth
    from traceweaver_b200.batch import build_batch_from_blocks
    blocks = synth.hotel_stream(4300, 24, seed=41) + [synth.make_block("hotel_frontend", 3, 3000, 150.0, seed=42)]
    hb = build_batch_from_blocks(blocks)
    assert hb.n_problems > 4096
    prm, sc, o_st = _pass0(engine, hb)
    for und in (None, sc):                                   # whole services / units between strong cuts
        _equal_oracle(_stitch(engine, prm, sc, und), o_st)


def test_one_block_grid_equals_default_grid(engine):
    """Two warps take every unit: long services of many units, one whose taken bitmap (> 256 words) lives
    in global memory, and short services of E = 2 and 3.  Assignments, ranks, candidate counts and the
    per-service counters (added up over a service's units) equal those of the default grid."""
    from traceweaver_b200 import synth
    from traceweaver_b200.batch import build_batch_from_blocks
    hb = build_batch_from_blocks([synth.make_block("hotel_frontend", 1, 5000, 100.0, seed=51),
                                  synth.make_block("hotel_search", 2, 2500, 150.0, seed=52),
                                  synth.make_block("hotel_frontend", 6, 200, 50.0, seed=53),
                                  synth.make_block("hotel_search", 6, 200, 125.0, seed=54)])
    prm, sc, o_st = _pass0(engine, hb)
    lib, h = engine.lib, engine.h
    default_grid = lib.tw_debug_stitch_grid(h, 0)
    assert default_grid > 1
    try:
        for und in (None, sc):
            ref = _stitch(engine, prm, sc, und)
            _equal_oracle(ref, o_st)
            assert lib.tw_debug_stitch_grid(h, 1) == 1
            one = _stitch(engine, prm, sc, und)
            assert lib.tw_debug_stitch_grid(h, 0) == default_grid
            for k in KEYS:
                assert np.array_equal(one[k], ref[k]), (k, und is None)
        assert lib.tw_debug_stitch_grid(h, default_grid + 1) < 0      # beyond the tables the bind reserved
    finally:
        lib.tw_debug_stitch_grid(h, 0)
