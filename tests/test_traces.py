"""Request trees (traces.py) on the host, without a GPU.

Two-tier synthetic deployments (synth.hotel_tree: frontend -> search, reservation, profile; search -> geo,
rate) are written as Jaeger JSON trace directories in the "hotel" layout (spans as recorded, server spans
referencing client spans) and the "node" layout (server spans only, referencing the caller's server span;
the loader synthesises the client twins), and read back with the loader.  Joined along the ground truth,
every reconstructed request must be exactly the batch nodes of one trace.  Crafted inputs cover the
detached fragment, the cycle and the malformed links."""
import json
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ALIBABA_DIR = os.path.join(HERE, "golden", "alibaba_synth")

# callee names per tier, in the call order of synth.hotel_tree
FRONT_CALLS = ("search", "reservation", "profile")
SEARCH_CALLS = ("geo", "rate")


def _request_spans(tree, s, r):
    """The spans of request r of replica s as (name, start, end, parent name) from the generator's arrays."""
    front, search = tree["blocks"]
    n = front.in_start.shape[1]
    sk = int(np.flatnonzero(tree["in_request"][front.in_start.size:][s * n:(s + 1) * n] == s * n + r)[0])
    t = lambda blk, e, i: (int(blk.out_start[e][s, int(blk.truth[e, s, i])]), int(blk.out_end[e][s, int(blk.truth[e, s, i])]))
    spans = [("frontend", int(front.in_start[s, r]), int(front.in_end[s, r]), None)]
    for e, name in enumerate(FRONT_CALLS):
        spans.append((name, *t(front, e, r), "frontend"))
    for e, name in enumerate(SEARCH_CALLS):
        spans.append((name, *t(search, e, sk), "search"))
    return spans, (int(search.in_start[s, sk]), int(search.in_end[s, sk]))


def write_tree_dir(tree, directory, layout, replica=0, n_req=None):
    """One Jaeger trace file per request of one replica of synth.hotel_tree.  "hotel": a client span in the
    caller's process and a server span (inside it) in the callee's, the server referencing the client;
    "node": only server spans, each referencing its caller's server span (the root "init-span" is recorded
    as a client span, as nodejs_microservices records it)."""
    front = tree["blocks"][0]
    n = front.in_start.shape[1] if n_req is None else n_req
    kind = lambda v: [{"key": "span.kind", "type": "string", "value": v}]
    names = ("frontend", "search") + FRONT_CALLS[1:] + SEARCH_CALLS
    procs = {f"p{k}": {"serviceName": nm, "tags": []} for k, nm in enumerate(names)}
    pid = {nm: f"p{k}" for k, nm in enumerate(names)}
    root_op = "HTTP GET /hotels" if layout == "hotel" else "init-span"
    for r in range(n):
        tid = f"{r:016x}"
        ref = lambda sid: [{"refType": "CHILD_OF", "traceID": tid, "spanID": sid}]
        span = lambda sid, op, st, en, k, proc, refs: {"traceID": tid, "spanID": sid, "operationName": op,
                                                        "references": refs, "startTime": st, "duration": en - st,
                                                        "tags": kind(k), "processID": pid[proc]}
        spans_, (ss, se) = _request_spans(tree, replica, r)
        (_, fs, fe, _), calls = spans_[0], spans_[1:]
        out = [span("root", root_op, fs, fe, "server" if layout == "hotel" else "client", "frontend", [])]
        for name, st, en, caller in calls:
            caller_sid = "root" if caller == "frontend" else ("s_search" if layout == "node" else "srv_search")
            if layout == "hotel":
                out.append(span(f"c_{name}", f"/{name}", st, en, "client", caller, ref(caller_sid)))
                a, b = (ss, se) if name == "search" else (st + 1, en - 1)
                out.append(span(f"srv_{name}", f"/{name}", a, b, "server", name, ref(f"c_{name}")))
            else:
                a, b = (ss, se) if name == "search" else (st, en)
                out.append(span(f"s_{name}", f"/{name}", a, b, "server", name, ref(caller_sid)))
        out.reverse()                                      # JSON order is not the call order
        with open(os.path.join(directory, f"{n - r:05d}.json"), "w") as fh:
            json.dump({"data": [{"traceID": tid, "spans": out, "processes": procs}]}, fh)


def _tree_dir(tmp_path, layout, n_req=150, seed=5):
    from traceweaver_b200 import synth
    tree = synth.hotel_tree(1, n_req, 120.0, seed=seed)
    d = tmp_path / layout
    d.mkdir()
    write_tree_dir(tree, str(d), layout)
    return str(d)


def load_batch(directory, layout):
    """services, batch, caller links, truth assignment and the trace id of every node."""
    from traceweaver_b200 import traces
    from traceweaver_b200.loader import load_jaeger_dir, to_host_batch
    services = [s for s in load_jaeger_dir(directory, layout=layout) if s.problem.in_accelerated_regime()]
    hb = to_host_batch(services)
    in_caller = traces.caller_links(services, hb)
    truth = np.concatenate([s.truth.reshape(-1) for s in services]).astype(np.int32)
    tid = [t for s in services for t, _ in s.in_ids]
    tid += [t for s in services for ids in s.out_ids for t, _ in ids]
    return services, hb, in_caller, truth, np.asarray(tid)


def check_one_tree_per_trace(root, size, tid, n_in):
    """Every root is an in-span; its nodes are exactly the nodes of one trace; every trace has one root."""
    assert (root >= 0).all(), "a cycle under the truth"
    roots = np.unique(root)
    assert (roots < n_in).all(), "a detached fragment under the truth"
    assert len(roots) == len(np.unique(tid))
    for r in roots:
        members = np.flatnonzero(root == r)
        assert size[r] == len(members)
        assert set(tid[members]) == {tid[r]}
        assert (tid == tid[r]).sum() == len(members)


@pytest.mark.parametrize("layout", ["hotel", "node"])
def test_truth_join_rebuilds_every_trace(tmp_path, layout):
    from traceweaver_b200.traces import assemble_host
    services, hb, in_caller, truth, tid = load_batch(_tree_dir(tmp_path, layout), layout)
    assert [s.name for s in services] == ["frontend", "search"]
    parent, root, size = assemble_host(hb, truth, in_caller)
    n_in = int(hb.prob_in_off[-1])
    check_one_tree_per_trace(root, size, tid, n_in)
    assert (size[np.unique(root)] == 7).all()             # frontend, its three calls, search and its two calls
    assert (in_caller[:150] == -1).all() and (in_caller[150:] >= n_in).all()


def test_truth_join_rebuilds_alibaba_traces():
    from traceweaver_b200.traces import assemble_host
    services, hb, in_caller, truth, tid = load_batch(ALIBABA_DIR, "alibaba")
    parent, root, size = assemble_host(hb, truth, in_caller)
    check_one_tree_per_trace(root, size, tid, int(hb.prob_in_off[-1]))


def _json_refs(directory):
    refs = {}
    for f in os.listdir(directory):
        for d in json.load(open(os.path.join(directory, f)))["data"]:
            for s in d["spans"]:
                refs[(s["traceID"], s["spanID"], s["tags"][-1]["value"])] = \
                    s["references"][0]["spanID"] if s["references"] else None
    return refs


@pytest.mark.parametrize("layout", ["hotel", "node", "alibaba"])
def test_caller_ids_follow_the_json_references(tmp_path, layout):
    from traceweaver_b200.loader import load_jaeger_dir
    directory = ALIBABA_DIR if layout == "alibaba" else _tree_dir(tmp_path, layout)
    refs = _json_refs(directory)
    services = load_jaeger_dir(directory, layout=layout)
    n_linked = 0
    for s in services:
        assert len(s.in_caller_ids) == s.problem.n_in
        for (t, sid), cid in zip(s.in_ids, s.in_caller_ids):
            if layout == "hotel":                           # the client span the server span references
                ref = refs[(t, sid, "server")]
                want = None if ref is None else (t, ref)
            elif layout == "node":                          # the client twin FixSpans gives every server span
                want = None if sid == "root" else (t, sid + "_client")
            else:                                           # the client record of the same rpc id
                want = None if refs[(t, sid, "server")] is None else (t, sid + ".client")
            assert cid == want, (s.name, sid)
            n_linked += cid is not None
    assert n_linked > 0


def _two_in_spans():
    from traceweaver_b200.batch import Problem, build_batch
    t = np.array([100, 200], np.int64)
    return build_batch([Problem(in_start=t, in_end=t + 50, out_start=[t + 10], out_end=[t + 20], preds=[[]])])


def test_unclaimed_out_span_is_a_detached_root():
    from traceweaver_b200.traces import assemble_host
    parent, root, size = assemble_host(_two_in_spans(), [0, -1], [-1, -1])   # nodes: in 0, 1; out 2, 3
    assert parent.tolist() == [-1, -1, 0, -1]
    assert root.tolist() == [0, 1, 0, 3]
    assert size.tolist() == [2, 1, 0, 1]


def test_link_cycle_has_no_root():
    from traceweaver_b200.traces import assemble_host
    # in-span 0 is the server side of out-span node 2, which the assignment gives to in-span 0
    parent, root, size = assemble_host(_two_in_spans(), [0, 1], [2, -1])
    assert parent.tolist() == [2, -1, 0, 1]
    assert root.tolist() == [-1, 1, -1, 1]
    assert size.tolist() == [0, 2, 0, 0]


@pytest.mark.parametrize("assign,in_caller,msg", [([0, 0], [-1, -1], "out-span node 2 is the child of two"),
                                                  ([0, 1], [3, 3], "out-span node 3 is the caller of two"),
                                                  ([0, 2], [-1, -1], "in-span node 1 has a child index outside"),
                                                  ([0, 1], [-1, 1], "in-span node 1 has a caller that is not")])
def test_malformed_links_raise(assign, in_caller, msg):
    from traceweaver_b200.traces import assemble_host
    with pytest.raises(ValueError, match=msg):
        assemble_host(_two_in_spans(), assign, in_caller)


def test_generated_tree_joins_to_requests():
    from traceweaver_b200 import synth
    from traceweaver_b200.traces import assemble_host
    tree = synth.hotel_tree(3, 200, 150.0, seed=2)
    hb = tree["hb"]
    n_in = int(hb.prob_in_off[-1])
    parent, root, size = assemble_host(hb, tree["truth"], tree["in_caller"])
    assert (root >= 0).all() and (root < 600).all()        # every node under a frontend in-span
    assert (size[:600] == 7).all()
    assert np.array_equal(tree["in_request"][root[:n_in]], tree["in_request"])


@pytest.mark.gpu
def test_device_join_converts_int64_links():
    """traces.assemble reads int64 assign / in_caller tensors as the int32 ones: the same join."""
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test needs a CUDA device")
    from traceweaver_b200 import synth, traces
    from traceweaver_b200.api import BatchSolver
    tree = synth.hotel_tree(3, 200, 150.0, seed=2)
    solver = BatchSolver(device=0, seed_select=10)
    try:
        eng = solver.engine
        assign = torch.from_numpy(np.asarray(tree["truth"], np.int32)).to(eng.device)
        in_caller = torch.from_numpy(np.asarray(tree["in_caller"], np.int32)).to(eng.device)
        want = traces.assemble(eng, tree["hb"], assign, in_caller)
        got = traces.assemble(eng, tree["hb"], assign.long(), in_caller.long())
        for k in ("parent", "root", "size"):
            assert torch.equal(got[k], want[k]), k
    finally:
        solver.close()
