"""tw_assemble_traces on the GPU against traces.assemble_host, element for element, on the truth and on
solve() results; the exact requests against truth.accuracy's end-to-end accuracy; malformed links, the
link cycle and the round bound; solve() untouched by a later assemble."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def solver():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test needs a CUDA device")
    from traceweaver_b200.api import BatchSolver
    s = BatchSolver(device=0, seed_select=10)
    s.engine.lib.tw_debug_trace_rounds.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    yield s
    s.close()


def _rounds(engine):
    launched, run = C.c_int(0), C.c_int(0)
    assert engine.lib.tw_debug_trace_rounds(engine.h, C.byref(launched), C.byref(run)) == 0
    return launched.value, run.value


def _same_as_host(solver, hb, assign, in_caller):
    from traceweaver_b200.traces import assemble_host
    got = solver.assemble(hb, assign, in_caller)
    parent, root, size = assemble_host(hb, assign, in_caller)
    assert np.array_equal(got["parent"], parent)
    assert np.array_equal(got["root"], root)
    assert np.array_equal(got["size"], size)
    return got


def _exact_share(solver, hb, assign, in_caller, truth, in_trace):
    """The share of exact requests and truth.accuracy's end-to-end accuracy, both over the requests whose
    in-spans all hang under one root of the truth join (all of them here: asserted)."""
    from traceweaver_b200 import truth as dev_truth
    from traceweaver_b200.traces import assemble_host
    eng = solver.engine
    _, root_true, _ = assemble_host(hb, truth, in_caller)
    n_in = int(hb.prob_in_off[-1])
    pairs = np.unique(np.stack([in_trace.astype(np.int64), root_true[:n_in].astype(np.int64)]), axis=1)
    assert pairs.shape[1] == len(np.unique(in_trace))      # one root per trace
    out = solver.assemble(hb, assign, in_caller, truth=truth)
    exact = out["exact"]
    share = (exact == 1).sum() / (exact >= 0).sum()
    assert (exact >= 0).sum() == len(np.unique(in_trace))
    tl = dev_truth.TraceLists.from_host_batch(hb, in_trace, int(in_trace.max()) + 1)
    import torch
    dev = eng.device
    acc = dev_truth.accuracy(eng, tl, torch.from_numpy(truth).to(dev), torch.from_numpy(np.asarray(assign, np.int32)).to(dev))
    assert share == acc["e2e_accuracy"], (share, acc["e2e_accuracy"])
    return share


@pytest.mark.parametrize("layout", ["hotel", "node", "alibaba"])
def test_device_join_equals_host_on_trace_directories(solver, tmp_path, layout):
    from test_traces import ALIBABA_DIR, _tree_dir, load_batch
    directory = ALIBABA_DIR if layout == "alibaba" else _tree_dir(tmp_path, layout, n_req=300)
    services, hb, in_caller, truth, tid = load_batch(directory, layout)
    _same_as_host(solver, hb, truth, in_caller)
    out = solver.solve(hb)
    assign = np.array(out["assign"])
    _same_as_host(solver, hb, assign, in_caller)
    in_trace = np.unique(tid[:int(hb.prob_in_off[-1])], return_inverse=True)[1].astype(np.int32)
    share = _exact_share(solver, hb, assign, in_caller, truth, in_trace)
    assert 0.0 < share <= 1.0


def test_device_join_on_a_batch_solve_splits(solver):
    from traceweaver_b200 import synth
    tree = synth.hotel_tree(560, 1000, 100.0, seed=31)
    hb = tree["hb"]
    assert int(hb.prob_in_off[-1]) > 1 << 20
    out = solver.solve(hb)
    assert solver.last_chunks > 1
    assign = np.array(out["assign"])
    got = _same_as_host(solver, hb, tree["truth"], tree["in_caller"])
    assert (got["size"][:560 * 1000] == 7).all()
    _same_as_host(solver, hb, assign, tree["in_caller"])
    share = _exact_share(solver, hb, assign, tree["in_caller"], tree["truth"], tree["in_request"])
    assert share > 0.5
    launched, run = _rounds(solver.engine)
    assert launched == int(np.ceil(np.log2(got["parent"].size))) + 1 and run < launched


def _two_in_spans():
    from test_traces import _two_in_spans as make
    return make()


def test_malformed_links_return_invalid(solver):
    from traceweaver_b200 import _abi
    for assign, in_caller, msg in [([0, 0], [-1, -1], "out-span node 2 is the child of two"),
                                   ([0, 1], [3, 3], "out-span node 3 is the caller of two"),
                                   ([0, 2], [-1, -1], "in-span node 1 has a child index outside"),
                                   ([0, 1], [-1, 1], "in-span node 1 has a caller that is not")]:
        with pytest.raises(_abi.TwError) as ex:
            solver.assemble(_two_in_spans(), assign, in_caller)
        assert ex.value.code == _abi.TW_ERR_INVALID and msg in str(ex.value)


def test_link_cycle_terminates_without_a_root(solver):
    eng = solver.engine
    before = eng.launch_count()
    got = _same_as_host(solver, _two_in_spans(), [0, 1], [2, -1])
    assert got["root"].tolist() == [-1, 1, -1, 1]
    launched, run = _rounds(eng)
    assert launched == 3                                   # ceil(log2 4) + 1
    assert eng.launch_count() - before == launched + 3     # two link kernels, the rounds, the roots
    assert _same_as_host(solver, _two_in_spans(), [0, -1], [-1, -1])["size"].tolist() == [2, 1, 0, 1]


def test_solve_unchanged_by_assemble(solver):
    from traceweaver_b200 import synth
    tree = synth.hotel_tree(8, 400, 120.0, seed=4)
    hb = tree["hb"]
    keys = ("assign", "topk_idx", "topk_cnt", "n_cand", "counters", "mis_rank")
    first = {k: np.array(v) for k, v in solver.solve(hb).items() if k in keys}
    n0 = solver.engine.launch_count()
    solver.solve(hb)
    per_solve = solver.engine.launch_count() - n0
    solver.assemble(hb, first["assign"], tree["in_caller"], truth=tree["truth"])
    n1 = solver.engine.launch_count()
    again = solver.solve(hb)
    assert solver.engine.launch_count() - n1 == per_solve
    for k in keys:
        assert np.array(again[k]).tobytes() == first[k].tobytes(), k
