"""tw_request_confidence on the GPU against traces.request_confidence_host and the CPU build of the device step,
element for element and bit for bit, on the truth and on solve() results (trace directories, a batch solve()
splits into groups, a time-compressed float64 batch); the roots against tw_assemble_traces; malformed links and
wrong sizes; run-to-run identity; solve() untouched by a later request_confidence."""
import numpy as np
import pytest

import emul_backend
from test_request_confidence import KEYS, check_same

pytestmark = pytest.mark.gpu
DEV_KEYS = tuple(k for k in KEYS if k != "q")


@pytest.fixture(scope="module")
def solver():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test needs a CUDA device")
    from traceweaver_b200.api import BatchSolver
    s = BatchSolver(device=0, seed_select=10)
    yield s
    s.close()


def _solved(solver, hb):
    out = solver.solve(hb, want_likelihood=True, want_scores=True, want_mixtures=True)
    return {k: np.array(v) for k, v in out.items()}


def _truth_out(solver, hb, truth, out):
    sc = solver.score(hb, truth, out["mixtures"])
    return dict(assign=np.asarray(truth, np.int32), chosen_score=sc["score"], chosen_code=sc["code"],
                topk_score=out["topk_score"], topk_idx=out["topk_idx"], topk_cnt=out["topk_cnt"])


def _same_everywhere(solver, hb, out, in_caller):
    from traceweaver_b200.traces import request_confidence_host
    got = solver.request_confidence(hb, out, in_caller)
    topk = {k: out[k] for k in ("topk_score", "topk_idx", "topk_cnt")}
    want = request_confidence_host(hb, out["assign"], in_caller, out["chosen_score"], out["chosen_code"], topk)
    got_arrays = dict(got, requests=np.array([got["requests"]], np.int32),
                      expected_exact=np.array([got["expected_exact"]]))
    check_same(got_arrays, want, keys=DEV_KEYS + ("root",))
    n_in = int(hb.prob_in_off[-1])
    cpu, rc = emul_backend.request_confidence(hb, out["assign"], got["root"][:n_in], out["chosen_score"],
                                              out["chosen_code"], topk)
    assert rc == 0
    check_same(got_arrays, cpu, keys=DEV_KEYS)
    asm = solver.assemble(hb, out["assign"], in_caller)
    assert np.array_equal(got["root"], asm["root"])
    assert np.array_equal(got["request"], np.flatnonzero(asm["root"][:n_in] == np.arange(n_in)))
    assert got["requests"] == len(got["request"])
    r = asm["root"][:n_in]
    mine = (r >= 0) & (r < n_in)
    assert np.array_equal(got["decisions"], np.bincount(r[mine], minlength=n_in))
    w = got["weakest"][got["request"]]
    assert (asm["root"][w] == got["request"]).all()
    return got


@pytest.mark.parametrize("layout", ["hotel", "node", "alibaba"])
def test_device_equals_host_on_trace_directories(solver, tmp_path, layout):
    from test_traces import ALIBABA_DIR, _tree_dir, load_batch
    directory = ALIBABA_DIR if layout == "alibaba" else _tree_dir(tmp_path, layout, n_req=300)
    _, hb, in_caller, truth, _ = load_batch(directory, layout)
    out = _solved(solver, hb)
    _same_everywhere(solver, hb, out, in_caller)
    _same_everywhere(solver, hb, _truth_out(solver, hb, truth, out), in_caller)


def test_device_equals_host_on_a_batch_solve_splits(solver):
    from traceweaver_b200 import synth
    tree = synth.hotel_tree(560, 1000, 100.0, seed=31)
    hb = tree["hb"]
    assert int(hb.prob_in_off[-1]) > 1 << 20
    out = _solved(solver, hb)
    assert solver.last_chunks > 1
    got = _same_everywhere(solver, hb, out, tree["in_caller"])
    assert got["requests"] == 560 * 1000
    _same_everywhere(solver, hb, _truth_out(solver, hb, tree["truth"], out), tree["in_caller"])


def test_device_equals_host_on_float64_times(solver):
    from test_critical_path import compressed
    from traceweaver_b200 import synth
    tree = synth.hotel_tree(4, 300, 120.0, seed=8)
    hf = compressed(tree["hb"], 7)
    assert hf.float_times
    _same_everywhere(solver, hf, _solved(solver, hf), tree["in_caller"])


def test_two_calls_are_byte_identical(solver):
    from traceweaver_b200 import synth
    tree = synth.hotel_tree(64, 1000, 120.0, seed=9)
    hb = tree["hb"]
    out = _solved(solver, hb)
    first = solver.request_confidence(hb, out, tree["in_caller"])
    again = solver.request_confidence(hb, out, tree["in_caller"])
    for k, v in first.items():
        assert np.asarray(again[k]).tobytes() == np.asarray(v).tobytes(), k


def test_malformed_links_and_wrong_sizes(solver):
    from test_traces import _two_in_spans
    from traceweaver_b200 import _abi
    hb = _two_in_spans()
    out = dict(assign=np.array([0, 1], np.int32), chosen_score=np.array([-1.0, -1.0]),
               chosen_code=np.zeros(2, np.uint8), topk_score=np.full((2, 5), np.nan),
               topk_idx=np.full(10, -1, np.int32), topk_cnt=np.zeros(2, np.uint8))
    for assign, in_caller, msg in [([0, 0], [-1, -1], "out-span node 2 is the child of two"),
                                   ([0, 1], [3, 3], "out-span node 3 is the caller of two"),
                                   ([0, 2], [-1, -1], "in-span node 1 has a child index outside"),
                                   ([0, 1], [-1, 1], "in-span node 1 has a caller that is not")]:
        with pytest.raises(_abi.TwError) as ex:
            solver.request_confidence(hb, dict(out, assign=np.array(assign, np.int32)), in_caller)
        assert ex.value.code == _abi.TW_ERR_INVALID and msg in str(ex.value)
        assert "tw_request_confidence" in str(ex.value)
    with pytest.raises(ValueError, match="topk_idx"):
        solver.request_confidence(hb, dict(out, topk_idx=np.zeros(4, np.int32)), [-1, -1])
    with pytest.raises(ValueError, match="score must have 2 entries"):
        solver.request_confidence(hb, dict(out, chosen_score=np.zeros(3)), [-1, -1])
    with pytest.raises(ValueError, match="want_likelihood=True"):
        solver.request_confidence(hb, {k: v for k, v in out.items() if k != "chosen_code"}, [-1, -1])
    with pytest.raises(ValueError, match="want_scores=True"):
        solver.request_confidence(hb, {k: v for k, v in out.items() if k != "topk_score"}, [-1, -1])


def test_solve_unchanged_by_request_confidence(solver):
    from traceweaver_b200 import synth
    tree = synth.hotel_tree(8, 400, 120.0, seed=4)
    hb = tree["hb"]
    first = _solved(solver, hb)
    n0 = solver.engine.launch_count()
    _solved(solver, hb)
    per_solve = solver.engine.launch_count() - n0
    solver.request_confidence(hb, first, tree["in_caller"])
    n1 = solver.engine.launch_count()
    again = _solved(solver, hb)
    assert solver.engine.launch_count() - n1 == per_solve
    for k, v in first.items():
        assert np.asarray(again[k]).tobytes() == np.asarray(v).tobytes(), k
