"""Critical paths (traces.critical_paths_host and the per-node steps of tw_core.cuh stepped on the CPU), without
a GPU.

Hand-built batches check each rule of the definition in traces.py: sequential calls; parallel calls with the
overlapping, truncated and nested call; children that start before or end after their parent; zero-length
children; the callee-position tie; a callee inside and outside the batch; negative durations; a cycle; a
detached fragment.  On synth.hotel_tree's truth every node is on the path and its self time has a closed form.
On the trace directories of test_traces the self times of every request add up to its latency.  The CPU build
of the device steps (tests/emul/tw_emul_critical.cpp, through emul_backend) must give the host reference's
arrays on all of them, with int64 times and with float64 times divided by 3 and 7."""
import ctypes as C

import numpy as np
import pytest

import emul_backend
from traceweaver_b200 import _abi
from traceweaver_b200.batch import HostBatch, Problem, build_batch

NODE_KEYS = ("root", "on_path", "self_us", "culprit")
SUM_KEYS = ("server_us", "server_visits", "call_us", "requests")


def compressed(hb, cf):
    """The batch with float64 times divided by cf (a time-compressed batch)."""
    arrays = dict(hb.arrays)
    for k in ("in_start", "in_end", "out_start", "out_end"):
        arrays[k] = np.asarray(hb.arrays[k], np.int64).astype(np.float64) / cf
    return HostBatch(problems=hb.problems, arrays=arrays)


def check_same(got, want, exact_sums):
    for k in NODE_KEYS:
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).astype(np.asarray(got[k]).dtype).tobytes(), k
    for k in ("server_visits", "requests"):
        assert np.array_equal(got[k], want[k]), k
    for k in ("server_us", "call_us"):
        if exact_sums:
            assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), k
        else:
            np.testing.assert_allclose(got[k], want[k], rtol=1e-9, atol=0, err_msg=k)


def check_invariant(res, hb, exact):
    """Per request: the self times of its on-path nodes add up to its latency."""
    root, on, self_us = res["root"], res["on_path"] == 1, res["self_us"]
    n_in = int(hb.prob_in_off[-1])
    req = np.flatnonzero(root[:n_in] == np.arange(n_in))
    total = np.zeros(len(root))
    np.add.at(total, root[on], self_us[on])
    got = total[req]
    if exact:
        assert np.array_equal(got, res["latency"])
    else:
        np.testing.assert_allclose(got, res["latency"], rtol=1e-12, atol=1e-9)
    assert ((root[on] >= 0) & (root[on] < n_in)).all()            # on-path nodes belong to requests
    assert on[req].all()


def paths_everywhere(hb, assign, in_caller, slow_us=0.0):
    """Host reference, with the invariant; the CPU step equal to it, int64 and float64 / 3, / 7."""
    from traceweaver_b200.traces import critical_paths_host
    want = critical_paths_host(hb, assign, in_caller, slow_us)
    check_invariant(want, hb, exact=True)
    check_same(emul_backend.critical_paths(hb, assign, in_caller, want["root"], slow_us), want, exact_sums=True)
    for cf in (3, 7):
        hf = compressed(hb, cf)
        wf = critical_paths_host(hf, assign, in_caller, slow_us / cf)
        check_invariant(wf, hf, exact=False)
        check_same(emul_backend.critical_paths(hf, assign, in_caller, wf["root"], slow_us / cf), wf,
                   exact_sums=False)
    return want


# ------------------------------------------------------------------------------------------------
# hand-built requests: a root service with one in-span and one out-span per call; a callee service
# (one in-span, one call it does not make) for call 0 when `callee` is given
# ------------------------------------------------------------------------------------------------
def _request(root, calls, callee=None):
    t = lambda v: np.array([v], np.int64)
    probs = [Problem(in_start=t(root[0]), in_end=t(root[1]), out_start=[t(s) for s, _ in calls],
                     out_end=[t(e) for _, e in calls], preds=[[] for _ in calls])]
    E = len(calls)
    assign, in_caller = [0] * E, [-1]
    if callee is not None:
        probs.append(Problem(in_start=t(callee[0]), in_end=t(callee[1]), out_start=[t(0)], out_end=[t(0)], preds=[[]]))
        assign.append(-1)
        in_caller.append(2)                              # n_in = 2: out-span node 2 is call 0
    return build_batch(probs, validate=False), assign, in_caller


def _walk(root, calls, callee=None):
    hb, assign, in_caller = _request(root, calls, callee)
    res = paths_everywhere(hb, assign, in_caller)
    n_in = int(hb.prob_in_off[-1])
    return res, n_in


def test_sequential_calls_are_all_on_the_path():
    res, n_in = _walk((0, 100), [(10, 30), (40, 70), (75, 90)])
    assert res["on_path"].tolist() == [1, 1, 1, 1]
    assert res["self_us"].tolist() == [35.0, 20.0, 30.0, 15.0]
    assert res["culprit"].tolist() == [0]
    assert res["latency"].tolist() == [100.0]


def test_parallel_calls_last_to_finish_truncated_and_nested():
    # B ends last; A was still running when B started (truncated to [10, 20]); C lies inside B
    res, _ = _walk((0, 100), [(10, 60), (20, 80), (30, 50)])
    assert res["on_path"].tolist() == [1, 1, 1, 0]
    assert res["self_us"].tolist() == [30.0, 10.0, 60.0, 0.0]
    assert res["culprit"].tolist() == [2]
    assert res["server_visits"].tolist() == [[1, 1]]
    assert res["call_us"].tolist() == [[10.0, 10.0], [60.0, 60.0], [0.0, 0.0]]


def test_children_beyond_their_parent_are_clipped():
    res, _ = _walk((0, 100), [(-10, 50), (60, 120)])
    assert res["self_us"].tolist() == [10.0, 50.0, 40.0]


def test_zero_length_and_outside_children_are_off_the_path():
    res, _ = _walk((0, 100), [(50, 50), (150, 160), (20, 30)])
    assert res["on_path"].tolist() == [1, 0, 0, 1]
    assert res["self_us"].tolist() == [90.0, 0.0, 0.0, 10.0]


def test_callee_position_breaks_a_tie():
    # both end at 80: callee 0 first; callee 1 was running when it started and is truncated to [20, 40]
    res, _ = _walk((0, 100), [(40, 80), (20, 80)])
    assert res["on_path"].tolist() == [1, 1, 1]
    assert res["self_us"].tolist() == [40.0, 40.0, 20.0]
    # callee 0 first again; callee 1 starts after it and is nested
    res, _ = _walk((0, 100), [(20, 80), (40, 80)])
    assert res["on_path"].tolist() == [1, 1, 0]
    assert res["self_us"].tolist() == [40.0, 60.0, 0.0]


def test_callee_inside_and_outside_the_batch():
    # call 0's server span is in the batch (clipped to the call), call 1's is not: all of it is call time
    res, n_in = _walk((0, 100), [(10, 30), (40, 90)], callee=(5, 25))
    assert n_in == 2
    # nodes: in 0 (root), in 1 (callee), out 2 (call 0), out 3 (call 1), out 4 (the callee's unmade call)
    assert res["on_path"].tolist() == [1, 1, 1, 1, 0]
    assert res["self_us"].tolist() == [30.0, 15.0, 5.0, 50.0, 0.0]
    assert res["culprit"].tolist() == [3, -1]
    assert res["server_us"].tolist() == [[30.0, 30.0], [15.0, 15.0]]
    assert res["server_visits"].tolist() == [[1, 1], [1, 1]]


def test_negative_durations_are_empty():
    res, _ = _walk((100, 40), [(50, 60)])              # a root that ends before it starts
    assert res["on_path"].tolist() == [1, 0]
    assert res["self_us"].tolist() == [0.0, 0.0]
    assert res["latency"].tolist() == [0.0]
    res, _ = _walk((0, 100), [(60, 40), (10, 20)])      # a call that ends before it starts
    assert res["on_path"].tolist() == [1, 0, 1]
    assert res["self_us"].tolist() == [90.0, 0.0, 10.0]


def test_cycle_and_detached_fragment_belong_to_no_request():
    from test_traces import _two_in_spans
    hb = _two_in_spans()                                 # in 0 [100, 150], in 1 [200, 250]; out 2, 3
    res = paths_everywhere(hb, [0, 1], [2, -1])    # in 0 and out 2 form a cycle
    assert res["root"].tolist() == [-1, 1, -1, 1]
    assert res["on_path"].tolist() == [0, 1, 0, 1]
    assert res["self_us"].tolist() == [0.0, 40.0, 0.0, 10.0]
    assert res["culprit"].tolist() == [-1, 1]
    assert res["requests"].tolist() == [1, 1]
    res = paths_everywhere(hb, [0, -1], [-1, -1])  # out 3 is a detached fragment
    assert res["on_path"].tolist() == [1, 1, 1, 0]
    assert res["requests"].tolist() == [2, 2]


def test_slow_column_takes_the_requests_at_or_above_the_threshold():
    from traceweaver_b200 import synth
    from traceweaver_b200.traces import critical_paths_host
    tree = synth.hotel_tree(2, 60, 120.0, seed=3)
    hb = tree["hb"]
    lat = critical_paths_host(hb, tree["truth"], tree["in_caller"], 0.0)["latency"]
    thr = float(np.sort(lat)[int(0.9 * (len(lat) - 1))])
    res = paths_everywhere(hb, tree["truth"], tree["in_caller"], thr)
    assert res["requests"].tolist() == [len(lat), int((lat >= thr).sum())]
    assert (res["server_visits"][:, 1] <= res["server_visits"][:, 0]).all()
    assert res["server_visits"][:, 1].sum() == 2 * int((lat >= thr).sum())


def test_generated_truth_puts_every_node_on_the_path():
    from traceweaver_b200 import synth
    tree = synth.hotel_tree(3, 200, 150.0, seed=2)
    hb = tree["hb"]
    res = paths_everywhere(hb, tree["truth"], tree["in_caller"])
    assert (res["on_path"] == 1).all()
    # closed form: the generator's calls are sequential and inside their caller, every server span inside
    # its client span, so a node's self time is its length less its children's
    n_in = int(hb.prob_in_off[-1])
    n = len(res["root"])
    start = np.concatenate([hb.in_start, hb.out_start]).astype(np.int64)
    end = np.concatenate([hb.in_end, hb.out_end]).astype(np.int64)
    from traceweaver_b200.traces import parents_host
    parent = parents_host(hb, tree["truth"], tree["in_caller"])
    child_len = np.zeros(n, np.int64)
    has = parent >= 0
    np.add.at(child_len, parent[has], (end - start)[has])
    assert np.array_equal(res["self_us"], (end - start - child_len).astype(np.float64))
    assert (res["culprit"][:600] >= 0).all() and (res["culprit"][600:] == -1).all()
    assert res["requests"].tolist() == [600, 600]


@pytest.mark.parametrize("layout", ["hotel", "node", "alibaba"])
def test_self_times_add_up_on_trace_directories(tmp_path, layout):
    from test_traces import ALIBABA_DIR, _tree_dir, load_batch
    directory = ALIBABA_DIR if layout == "alibaba" else _tree_dir(tmp_path, layout)
    services, hb, in_caller, truth, tid = load_batch(directory, layout)
    res = paths_everywhere(hb, truth, in_caller)
    assert res["requests"][0] == len(np.unique(tid))


def test_malformed_links_raise():
    from test_traces import _two_in_spans
    from traceweaver_b200.traces import critical_paths_host
    with pytest.raises(ValueError, match="out-span node 2 is the child of two"):
        critical_paths_host(_two_in_spans(), [0, 0], [-1, -1], 0.0)


def test_critical_out_layout():
    assert C.sizeof(_abi.TwCriticalOut) == 8 * 8
