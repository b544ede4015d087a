"""tw_assemble_traces and tw_critical_paths on the GPU on deep, irregular trees (tests/deep_tree_util.py),
against the host references (traces.assemble_host, traces.critical_paths_host).

The join on chains of 1 000 to 3 000 levels, caterpillars and random trees in every service order, and on
a deep tree under a long cycle.  The critical paths with the level count the join's rounds give and then
with every forced count 1 .. 64 (tw_debug_critical_force_levels): byte-identical every time, with no
engine error, on spine-last trees whose last level walks hundreds of levels; int64 and float64 times; the
natural level count and the launch count from the round hooks; culprit ties across levels."""
import contextlib
import ctypes as C

import numpy as np
import pytest

from deep_tree_util import ORDERS, deep_trees
from test_critical_path import compressed
from test_deep_trees import cycle_trees
from test_gpu_critical_path import _same_as_host

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def solver():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test needs a CUDA device")
    from traceweaver_b200.api import BatchSolver
    s = BatchSolver(device=0, seed_select=10)
    lib = s.engine.lib
    lib.tw_debug_trace_rounds.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.tw_debug_critical_levels.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    lib.tw_debug_critical_force_levels.argtypes = [C.c_void_p, C.c_int]
    yield s
    s.close()


def _rounds(solver):
    launched, run = C.c_int(0), C.c_int(0)
    assert solver.engine.lib.tw_debug_trace_rounds(solver.engine.h, C.byref(launched), C.byref(run)) == 0
    return launched.value, run.value


def _levels(solver):
    levels = C.c_int(0)
    assert solver.engine.lib.tw_debug_critical_levels(solver.engine.h, C.byref(levels)) == 0
    return levels.value


@contextlib.contextmanager
def _forced(solver, levels):
    eng = solver.engine
    assert eng.lib.tw_debug_critical_force_levels(eng.h, levels) == 0
    try:
        yield
    finally:
        assert eng.lib.tw_debug_critical_force_levels(eng.h, 0) == 0


def _same_at_every_level_count(solver, hb, assign, in_caller):
    """The natural level count against the host, then every forced count byte-identical to it."""
    natural = _same_as_host(solver, hb, assign, in_caller)
    for L in range(1, 65):
        with _forced(solver, L):
            got = solver.critical_paths(hb, assign, in_caller, slow_quantile=0.9)
            assert _levels(solver) == L
        for k, v in natural.items():
            assert np.asarray(got[k]).tobytes() == np.asarray(v).tobytes(), (L, k)
    return natural


def _assemble_equals_host(solver, g, in_caller=None):
    from traceweaver_b200.traces import assemble_host
    in_caller = g["in_caller"] if in_caller is None else in_caller
    got = solver.assemble(g["hb"], g["assign"], in_caller)
    want = dict(zip(("parent", "root", "size"), assemble_host(g["hb"], g["assign"], in_caller)))
    for k in ("parent", "root", "size"):
        assert np.array_equal(got[k], want[k]), k
    launched, run = _rounds(solver)
    assert 1 <= run <= launched
    return got


@pytest.mark.parametrize("order", ORDERS)
def test_join_on_deep_chains_caterpillars_and_random_trees(solver, order):
    for depth in (1000, 3000):
        g = deep_trees(depth, callees=1, requests=3, order=order, seed=depth)
        got = _assemble_equals_host(solver, g)
        assert (got["size"][g["roots"]] == 2 * depth).all()
    g = deep_trees(1500, callees=4, spine="last", requests=2, order=order, seed=2)
    _assemble_equals_host(solver, g)
    g = deep_trees(2000, callees=8, random_shape=True, requests=8, timing="mixed", order=order, seed=3)
    got = _assemble_equals_host(solver, g)
    assert (got["root"] >= 0).all()


def test_join_puts_a_deep_tree_under_a_long_cycle_in_no_request(solver):
    g = cycle_trees(1000)
    got = _assemble_equals_host(solver, g, g["in_caller"])
    assert (got["root"][g["lost"]] == -1).all()
    assert (np.delete(got["root"], g["lost"]) >= 0).all()


@pytest.mark.parametrize("depth", [20, 500])
def test_paths_are_the_same_at_every_level_count(solver, depth):
    g = deep_trees(depth, callees=8, spine="last", requests=3, seed=depth)
    got = _same_at_every_level_count(solver, g["hb"], g["assign"], g["in_caller"])
    assert (got["on_path"] == 1).all()
    slow = int((got["latency_us"] >= got["slow_us"]).sum())     # the slow column: at least the 0.9-quantile
    assert got["requests"].tolist() == [3, slow] and 0 < slow < 3


def test_paths_at_every_level_count_on_float64_times(solver):
    g = deep_trees(60, callees=6, spine="last", timing="mixed", requests=4, order="shuffled", seed=8)
    for cf in (3, 7):
        hf = compressed(g["hb"], cf)
        assert hf.float_times
        _same_at_every_level_count(solver, hf, g["assign"], g["in_caller"])


@pytest.mark.parametrize("order", ORDERS)
def test_paths_on_random_trees(solver, order):
    g = deep_trees(300, callees=8, random_shape=True, requests=10, timing="mixed", order=order, seed=11)
    _same_at_every_level_count(solver, g["hb"], g["assign"], g["in_caller"])


def test_deep_spine_last_tree_walks_without_error(solver):
    g = deep_trees(2000, callees=3, spine="last", requests=2, order="shuffled", seed=12)
    got = _same_as_host(solver, g["hb"], g["assign"], g["in_caller"])
    assert (got["on_path"] == 1).all()
    with _forced(solver, 1):
        again = solver.critical_paths(g["hb"], g["assign"], g["in_caller"], slow_quantile=0.9)
    for k, v in got.items():
        assert np.asarray(again[k]).tobytes() == np.asarray(v).tobytes(), k


def test_natural_level_count_and_launches_follow_the_rounds(solver):
    cases = [deep_trees(d, callees=c, spine="last", requests=2, order=o, seed=d)
             for d, c, o in ((1, 1, "root"), (2, 2, "leaf"), (5, 4, "shuffled"), (40, 2, "root"), (700, 2, "leaf"))]
    eng = solver.engine
    for g in cases:
        n0 = eng.launch_count()
        solver.critical_paths(g["hb"], g["assign"], g["in_caller"])
        launches = eng.launch_count() - n0
        launched, run = _rounds(solver)
        L = _levels(solver)
        assert L == (1 if run == 1 else min(64, 2 ** (run - 2) + 1)), (run, L)
        # the join (two link kernels, its rounds, the roots), the levels, two culprit kernels, the reduction
        assert launches == (3 + launched) + L + 3
        with _forced(solver, 7):
            n0 = eng.launch_count()
            solver.critical_paths(g["hb"], g["assign"], g["in_caller"])
            assert eng.launch_count() - n0 == (3 + launched) + 7 + 3
    # a cycle keeps every round moving: 64 levels, and the requests outside it equal to the host
    g = cycle_trees(200)
    got = _same_as_host(solver, g["hb"], g["assign"], g["in_caller"])
    launched, run = _rounds(solver)
    assert run == launched and _levels(solver) == 64
    assert (got["on_path"][g["lost"]] == 0).all() and got["requests"][0] == 1


def test_culprit_ties_across_levels_pick_the_smallest_node(solver):
    g = deep_trees(80, callees=4, spine="last", requests=3, order="shuffled", const_times=True, seed=13)
    got = _same_at_every_level_count(solver, g["hb"], g["assign"], g["in_caller"])
    on, self_us, root = got["on_path"] == 1, got["self_us"], got["root"]
    for r in g["roots"]:
        mine = np.flatnonzero(on & (root == r))
        top = mine[self_us[mine] == self_us[mine].max()]
        assert len(top) > 80
        assert got["culprit"][r] == top.min()


def test_force_levels_hook_checks_its_range_and_later_calls_start_clean(solver):
    from traceweaver_b200 import _abi
    eng = solver.engine
    for bad in (-1, 65, 1000):
        assert eng.lib.tw_debug_critical_force_levels(eng.h, bad) == _abi.TW_ERR_INVALID
    g = deep_trees(30, callees=8, spine="last", requests=2, seed=14)
    first = _same_as_host(solver, g["hb"], g["assign"], g["in_caller"])
    natural = _levels(solver)
    with _forced(solver, 1):
        solver.critical_paths(g["hb"], g["assign"], g["in_caller"])
    eng.status()
    again = _same_as_host(solver, g["hb"], g["assign"], g["in_caller"])
    assert _levels(solver) == natural
    for k, v in first.items():
        assert np.asarray(again[k]).tobytes() == np.asarray(v).tobytes(), k
