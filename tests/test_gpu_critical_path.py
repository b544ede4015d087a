"""tw_critical_paths on the GPU against traces.critical_paths_host, element for element, on the truth and on
solve() results (trace directories, a batch solve() splits into groups, a time-compressed float64 batch); the
roots against tw_assemble_traces; malformed links; run-to-run identity; the launch count; solve() untouched by
a later critical_paths."""
import ctypes as C

import numpy as np
import pytest

from test_critical_path import check_same, compressed

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def solver():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test needs a CUDA device")
    from traceweaver_b200.api import BatchSolver
    s = BatchSolver(device=0, seed_select=10)
    s.engine.lib.tw_debug_trace_rounds.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    s.engine.lib.tw_debug_critical_levels.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    yield s
    s.close()


def _same_as_host(solver, hb, assign, in_caller, q=0.9):
    from traceweaver_b200.traces import critical_paths_host
    got = solver.critical_paths(hb, assign, in_caller, slow_quantile=q)
    want = critical_paths_host(hb, assign, in_caller, got["slow_us"])
    check_same(got, want, exact_sums=not hb.float_times)
    assert got["latency_us"].tobytes() == want["latency"].tobytes()
    assert np.array_equal(got["request"], np.flatnonzero(want["root"][:len(want["culprit"])] ==
                                                         np.arange(len(want["culprit"]))))
    assert np.array_equal(got["root"], solver.assemble(hb, assign, in_caller)["root"])
    lat = got["latency_us"]
    assert got["slow_us"] in lat and got["slow_us"] == np.sort(lat)[int(np.floor(q * (len(lat) - 1)))]
    return got


@pytest.mark.parametrize("layout", ["hotel", "node", "alibaba"])
def test_device_paths_equal_host_on_trace_directories(solver, tmp_path, layout):
    from test_traces import ALIBABA_DIR, _tree_dir, load_batch
    directory = ALIBABA_DIR if layout == "alibaba" else _tree_dir(tmp_path, layout, n_req=300)
    services, hb, in_caller, truth, tid = load_batch(directory, layout)
    got = _same_as_host(solver, hb, truth, in_caller)
    assert got["requests"][0] == len(np.unique(tid))
    _same_as_host(solver, hb, np.array(solver.solve(hb)["assign"]), in_caller)


def test_device_paths_on_a_batch_solve_splits(solver):
    from traceweaver_b200 import synth
    tree = synth.hotel_tree(560, 1000, 100.0, seed=31)
    hb = tree["hb"]
    assert int(hb.prob_in_off[-1]) > 1 << 20
    assign = np.array(solver.solve(hb)["assign"])
    assert solver.last_chunks > 1
    got = _same_as_host(solver, hb, tree["truth"], tree["in_caller"], q=0.99)
    assert (got["on_path"] == 1).all()
    _same_as_host(solver, hb, assign, tree["in_caller"], q=0.99)


def test_device_paths_on_float64_times(solver):
    from traceweaver_b200 import synth
    tree = synth.hotel_tree(4, 300, 120.0, seed=8)
    for cf in (3, 7):
        hf = compressed(tree["hb"], cf)
        assert hf.float_times
        _same_as_host(solver, hf, tree["truth"], tree["in_caller"])


def test_malformed_links_return_invalid(solver):
    from test_traces import _two_in_spans
    from traceweaver_b200 import _abi
    for assign, in_caller, msg in [([0, 0], [-1, -1], "out-span node 2 is the child of two"),
                                   ([0, 1], [3, 3], "out-span node 3 is the caller of two"),
                                   ([0, 2], [-1, -1], "in-span node 1 has a child index outside"),
                                   ([0, 1], [-1, 1], "in-span node 1 has a caller that is not")]:
        with pytest.raises(_abi.TwError) as ex:
            solver.critical_paths(_two_in_spans(), assign, in_caller)
        assert ex.value.code == _abi.TW_ERR_INVALID and msg in str(ex.value)
        assert "tw_critical_paths" in str(ex.value)


def test_two_calls_are_byte_identical_and_launches_are_counted(solver):
    from traceweaver_b200 import synth
    tree = synth.hotel_tree(64, 1000, 120.0, seed=9)
    hb = tree["hb"]
    eng = solver.engine
    first = solver.critical_paths(hb, tree["truth"], tree["in_caller"])
    n0 = eng.launch_count()
    again = solver.critical_paths(hb, tree["truth"], tree["in_caller"])
    launches = eng.launch_count() - n0
    for k, v in first.items():
        assert np.asarray(again[k]).tobytes() == np.asarray(v).tobytes(), k
    launched, run = C.c_int(0), C.c_int(0)
    eng.lib.tw_debug_trace_rounds(eng.h, C.byref(launched), C.byref(run))
    levels = C.c_int(0)
    eng.lib.tw_debug_critical_levels(eng.h, C.byref(levels))
    assert levels.value == 3                              # depth 4 links: rounds 0 and 1 move, round 2 does not
    # the join (two link kernels, its rounds, the roots), the levels, two culprit kernels, the reduction
    assert launches == (3 + launched.value) + levels.value + 3


def test_solve_unchanged_by_critical_paths(solver):
    from traceweaver_b200 import synth
    tree = synth.hotel_tree(8, 400, 120.0, seed=4)
    hb = tree["hb"]
    keys = ("assign", "topk_idx", "topk_cnt", "n_cand", "counters", "mis_rank")
    first = {k: np.array(v) for k, v in solver.solve(hb).items() if k in keys}
    n0 = solver.engine.launch_count()
    solver.solve(hb)
    per_solve = solver.engine.launch_count() - n0
    solver.critical_paths(hb, first["assign"], tree["in_caller"])
    n1 = solver.engine.launch_count()
    again = solver.solve(hb)
    assert solver.engine.launch_count() - n1 == per_solve
    for k in keys:
        assert np.array(again[k]).tobytes() == first[k].tobytes(), k
