"""Jaeger JSON traces -> SoA problems, without `Span` objects (SURVEY.md §8 row f-1).

The reference builds a `Span` object per JSON span, walks every trace tree, deep-copies the span
lists per service and partitions them by the service at the other end before it can call
`TraceWeaverV3.FindAssignments` (executor.py: ParseSpansJson :342-400, ParseJsonTrace :755-793,
ProcessTraceData :798-848, the per-service loop :1080-1140, utils.GetGroundTruth utils.py:22-32,
FindOrder executor.py:214-285).  This module restates that data path for two of the reference's
dataset layouts — "hotel": spans as recorded (`--fix 2` hotel_reservation, first span
"HTTP GET /hotels"; any dataset whose spans carry `span.kind` client/server tags), "media": the
FixSpans2 rewrite (`--fix 1` media_microservices, executor.py:539-640), "node": the FixSpans rewrite
(`--fix 0` nodejs_microservices, executor.py:511-537) — and emits, per solved service, exactly what
the engine binds:

    in_start / in_end            int64 [n]      the service's server spans, sorted by (start, end)
    out_start[e] / out_end[e]    int64 [n_e]    client spans per callee, same sort, callees in the
                                                topological order of the invocation graph
    preds[e]                     the DAG's in-edges (precedence constraints)
    truth[e, i]                  index of the true child in callee e's list (accuracy only)
    ids                          (trace id, span id) per row, to map results back

Same order-defining rules as the reference, because ties in `start` are broken by list order:
files by root start time (np.argsort, executor.py:305-309), spans of a trace in pre-order with
children sorted by start (:826-836), partitions stable-sorted by (start, end) (:1107), the trace
cap `cnt > 1000` (:873).  tests/test_loader.py checks the output against the goldens minted from
the reference's own loader (12 hotel + 6 media + 4 nodejs services: arrays, ids, graph, ground
truth equal).  `--fix 3` / `--fix 4` are the "hotel" layout with another `first_span` (no span
rewrite, executor.py:760-761; not checked against goldens — no such dataset is shipped).  Not built:
`--fix 5` (Alibaba: no first-span filter, self-loop rewriting, executor.py:386-400).
"""
import json
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

from .batch import Problem, build_batch

HOTEL_FIRST_SPAN = "HTTP GET /hotels"          # executor.py:759 (--fix 2)
MEDIA_FIRST_SPAN = "ComposeReview"             # executor.py:758 (--fix 1)
NODE_FIRST_SPAN = "init-span"                  # executor.py:757 (--fix 0)
MAX_TRACES = 1000                              # executor.py:873: stop once cnt > 1000


@dataclass
class ServiceProblem:
    """One solved service (`process`) of a trace directory."""
    name: str
    in_ep: str                       # the caller partition ("client_<op>" for the entry service)
    out_eps_given: List[str]         # callee order as the reference hands it to FindAssignments
    out_eps: List[str]               # topological order = ep index of the engine
    problem: Problem
    in_ids: List[tuple]
    out_ids: List[List[tuple]]       # per ep (topological order)
    truth: np.ndarray                # int32 [E, n], -1 where the trace has no such child
    graph_edges: List[tuple] = field(default_factory=list)
    # per in-span: (trace id, span id) of the client span of its RPC (the span it references, or the client
    # twin a rewrite gave it), None for a request that enters here.  The observed links of the request trees
    # (traces.caller_links); an id is a span reference, which names the trace as well as the span.
    in_caller_ids: List[Optional[tuple]] = field(default_factory=list)


def _span_kind(span):
    kind = None
    for tag in span["tags"]:                     # the LAST span.kind tag wins (executor.py:351-353)
        if tag["key"] == "span.kind":
            kind = tag["value"]
    return kind


def trace_files(directory: str) -> List[str]:
    """*.json files of the directory ordered by the start time of their root span
    (GetAllTracesInDir / TimeOrder, executor.py:287-339, without the pickle cache)."""
    files = [f for f in os.listdir(directory) if os.path.isfile(os.path.join(directory, f)) and f.endswith("json")]
    full = os.path.abspath(directory)
    files = [os.path.join(full, f) for f in files]
    starts = []
    for path in files:
        with open(path, "r") as fh:
            data = json.load(fh).get("data", [])
        t = float("inf")
        if data:
            root = next((s for s in data[0].get("spans", []) if len(s.get("references", [])) == 0), None)
            if root is not None:
                t = float(root["startTime"])
        starts.append(t)
    order = np.argsort(starts)
    return [files[i] for i in order]


class _Rows:
    """Growing SoA of one service's spans of one kind (server or client)."""

    def __init__(self):
        self.start, self.dur, self.tid, self.sid, self.other, self.caller = [], [], [], [], [], []

    def add(self, start, dur, tid, sid, other, caller=None):
        self.start.append(start)
        self.dur.append(dur)
        self.tid.append(tid)
        self.sid.append(sid)
        self.other.append(other)
        self.caller.append(caller)


def _nodes_plain(d, path):
    """Spans of one trace as the reference holds them after ParseSpansJson (no rewrite): dict order =
    JSON order.  node = [trace, sid, start, dur, op, service, kind, parent position or -1]."""
    spans = d["spans"]
    proc = {pid: p["serviceName"] for pid, p in d["processes"].items()}
    index = {s["spanID"]: k for k, s in enumerate(spans)}
    nodes = []
    for s in spans:
        if len(s["references"]) > 1:
            raise ValueError(f"{path}: span with several references (spans.py:41)")
        par = index[s["references"][0]["spanID"]] if s["references"] else -1
        nodes.append([s["traceID"], s["spanID"], s["startTime"], s["duration"], s["operationName"],
                      proc[s["processID"]], _span_kind(s), par])
    return nodes


def _nodes_node(d, path):
    """FixSpans (executor.py:511-537), the `--fix 0` rewrite of the nodejs_microservices traces: the
    root "init-span" (recorded as a client span) becomes a server span, every recorded server span
    gets a client twin with the same timing in its caller's process.  The reference looks the
    caller up in a static service table (executor.py:109-115); the parent span's own process is the
    same service in these traces.  Dict order: recorded spans, then the twins, both in JSON order."""
    spans = d["spans"]
    proc = {pid: p["serviceName"] for pid, p in d["processes"].items()}
    index = {s["spanID"]: k for k, s in enumerate(spans)}
    n = len(spans)
    nodes, twins = [], []
    for k, s in enumerate(spans):
        if len(s["references"]) > 1:
            raise ValueError(f"{path}: span with several references (spans.py:41)")
        kind = _span_kind(s)
        par = index[s["references"][0]["spanID"]] if s["references"] else -1
        base = [s["traceID"], s["spanID"], s["startTime"], s["duration"], s["operationName"], proc[s["processID"]]]
        if kind == "client":
            nodes.append(base + ["server", par])
        elif kind == "server":
            if par < 0:
                raise ValueError(f"{path}: server span without a parent (FixSpans indexes references[0])")
            twin_pos = n + len(twins)
            nodes.append(base + ["server", twin_pos])
            twins.append([s["traceID"], s["spanID"] + "_client", s["startTime"], s["duration"], s["operationName"],
                          proc[spans[par]["processID"]], "client", par])
        else:
            nodes.append(base + [kind, par])
    return nodes + twins


def _nodes_alibaba(d, path, loop_map):
    """The `--fix 5` reading of traces in the Alibaba ETL's layout (ParseSpansJson with first_span None,
    executor.py:377-470): every rpc is a server record (processID = callee) plus a client twin with the SAME
    spanID (processID = caller); there is no `processes` table (ParseProcessesJson2: the processID is the
    service).  The client twin's id gets the suffix ".client" and becomes the parent of its server record;
    an rpc whose caller equals its callee (a self loop) has its callee renamed to a fresh "...-loop" service —
    the reference draws a random name per RPC ID (`selfLoopMap` is keyed by the sanitised span id and lives
    across traces, executor.py:392-402); here the name is "<callee>-<n>-loop" — and every client span below
    a span whose rpc id is in that map is moved to its parent's service (executor.py:447-466).  A trace in
    which some child is not contained in its parent is dropped (executor.py:425-441): returns None."""
    spans = d["spans"]
    nodes, key_of = [], {}
    for s in spans:
        kind = _span_kind(s)
        sid = s["spanID"]
        refs = [r["spanID"] for r in s["references"]]
        if len(refs) > 1:
            raise ValueError(f"{path}: span with several references (spans.py:41)")
        if kind == "client":
            sid = sid + ".client"
        elif kind == "server" and len(refs) == 1:
            refs[0] = sid + ".client"
        service = s["processID"]
        if s["caller"] == s["callee"]:
            rpc = sid[:-7] if sid.endswith(".client") else sid
            if rpc not in loop_map:
                loop_map[rpc] = f"{s['callee']}-{len(loop_map)}-loop"
            if kind == "server":
                service = loop_map[rpc]
        key_of[sid] = len(nodes)
        nodes.append([s["traceID"], sid, s["startTime"], s["duration"], s.get("requestType", s.get("operationName")),
                      service, kind, refs[0] if refs else None])
    children = [[] for _ in nodes]
    for k, nd in enumerate(nodes):
        par = nd[7]
        nd[7] = key_of.get(par, -1) if par is not None else -1
        if par is not None and par in key_of:
            children[key_of[par]].append(k)
    root = next((k for k, nd in enumerate(nodes) if nd[7] < 0 and not spans[k]["references"]), None)
    if root is not None:
        stack = [root]
        while stack:                                     # check_time_constraints, executor.py:425-438
            k = stack.pop()
            for c in children[k]:
                if not (nodes[k][2] <= nodes[c][2] and nodes[k][2] + nodes[k][3] >= nodes[c][2] + nodes[c][3]):
                    return None
                stack.append(c)
        stack = [(root, False)]
        while stack:                                     # traverse_and_update / update_references, :447-466
            k, below_loop = stack.pop()
            sid = nodes[k][1]
            rpc = sid[:-7] if sid.endswith(".client") else sid
            below = below_loop or rpc in loop_map
            for c in children[k]:
                if below and nodes[c][6] == "client":
                    nodes[c][5] = nodes[k][5]
                stack.append((c, below))
    return nodes


def _nodes_media(d, path):
    """FixSpans2 (executor.py:539-640), the `--fix 1` rewrite of media_microservices traces, whose
    spans carry no span.kind: the "ComposeReview" span becomes the root (its ancestors are dropped,
    its id becomes the trace id), spans in the same process as their parent are dropped, every
    remaining span is a server span and gets a client twin with the same timing in its parent's
    process.  Dict order after the rewrite: stable sort by start of [servers in JSON order with the
    new root last, twins in the same order]."""
    spans = d["spans"]
    proc = {pid: p["serviceName"] for pid, p in d["processes"].items()}
    index = {s["spanID"]: k for k, s in enumerate(spans)}
    parent = [index[s["references"][0]["spanID"]] if s["references"] else -1 for s in spans]
    roots = [k for k, s in enumerate(spans) if s["operationName"] == MEDIA_FIRST_SPAN]
    if len(roots) != 1:
        raise ValueError(f"{path}: expected one {MEDIA_FIRST_SPAN} span")
    c = roots[0]
    dropped = set()
    k = parent[c]
    while k >= 0:                                                                        # DeleteAncestors
        dropped.add(k)
        k = parent[k]
    order = [k for k in range(len(spans)) if k not in dropped and k != c] + [c]
    for k in order:                                                                      # same-process children
        if k != c and parent[k] in dropped:
            raise ValueError(f"{path}: span hangs off a dropped ancestor (FixSpans2 would raise KeyError)")
    same = {k for k in order if k != c and spans[parent[k]]["processID"] == spans[k]["processID"]}
    keep = [k for k in order if k not in same]
    for k in keep:
        if k != c and parent[k] in same:
            raise ValueError(f"{path}: child of a dropped same-process span (FixSpans2 would raise KeyError)")
    tid = spans[c]["traceID"]
    servers, twins = [], []
    for k in keep:
        s = spans[k]
        sid = tid if k == c else s["spanID"]
        # parent position is patched below: a server's parent is its twin, a twin's parent the server
        servers.append([tid, sid, s["startTime"], s["duration"], s["operationName"], proc[s["processID"]], "server", k])
        if k != c:
            twins.append([tid, sid + "_client", s["startTime"], s["duration"], s["operationName"],
                          proc[spans[parent[k]]["processID"]], "client", k])
    merged = servers + twins
    merged_order = sorted(range(len(merged)), key=lambda q: merged[q][2])                # stable, by start
    pos_server = {}
    pos_twin = {}
    for newpos, q in enumerate(merged_order):
        node = merged[q]
        (pos_server if node[6] == "server" else pos_twin)[node[7]] = newpos
    nodes = []
    for q in merged_order:
        node = list(merged[q])
        k = node[7]
        if node[6] == "server":
            node[7] = -1 if k == c else pos_twin[k]
        else:
            node[7] = pos_server[parent[k]]
        nodes.append(node)
    return nodes


def load_jaeger_dir(directory: str, first_span: Optional[str] = HOTEL_FIRST_SPAN, max_traces: int = MAX_TRACES,
                    files: Optional[Sequence[str]] = None, layout: str = "hotel", engine=None) -> List[ServiceProblem]:
    """All solvable services of a trace directory, in the order the reference visits them.
    engine: a traceweaver_b200.engine.Engine -> the ground truth and FindOrder of all services are derived
    on the device in one batch (row f-2); None -> NumPy on the host (same result).
    layout "hotel": spans as recorded (`--fix 2`); "media": FixSpans2 rewrite (`--fix 1`, first span
    "ComposeReview"); "node": FixSpans rewrite (`--fix 0`, first span "init-span")."""
    if layout not in ("hotel", "media", "node", "alibaba"):
        raise ValueError(f"layout {layout!r}: hotel (--fix 2), media (--fix 1), node (--fix 0) and alibaba (--fix 5) are built")
    if layout == "alibaba":
        first_span = None                                # every rooted trace is taken (executor.py:765)
    loop_map: Dict[str, str] = {}
    if layout == "media":
        first_span = MEDIA_FIRST_SPAN
    if layout == "node":
        first_span = NODE_FIRST_SPAN
    files = list(files) if files is not None else trace_files(directory)
    ins: Dict[str, _Rows] = {}
    outs: Dict[str, _Rows] = {}
    cnt = 0
    for path in files:
        with open(path, "r") as fh:
            data = json.load(fh)["data"]
        accepted = []
        for d in data:
            spans = d["spans"]
            if any(s["traceID"] != spans[0]["traceID"] for s in spans):
                raise ValueError(f"{path}: different trace ids inside one trace")       # executor.py:372-374
            if layout == "media" or any(len(s["references"]) == 0 for s in spans):
                accepted.append(d)
        if len(accepted) != 1:
            raise ValueError(f"{path}: expected exactly one rooted trace (executor.py:790)")
        if layout == "alibaba":
            nodes = _nodes_alibaba(accepted[0], path, loop_map)
            if nodes is None:
                continue                                 # time constraint violated: the trace is skipped (:869-871)
        else:
            nodes = {"media": _nodes_media, "node": _nodes_node, "hotel": _nodes_plain}[layout](accepted[0], path)
        children: List[List[int]] = [[] for _ in nodes]
        root = None
        for k, node in enumerate(nodes):
            if node[7] < 0:
                root = k                                                                 # the last root wins (:822-823)
            else:
                children[node[7]].append(k)
        if first_span is not None and nodes[root][4] != first_span:
            continue
        for ch in children:
            ch.sort(key=lambda k: nodes[k][2])                                           # stable (:826-829)
        stack = [root]
        while stack:                                                                     # pre-order (:831-836)
            k = stack.pop()
            tid, sid, start, dur, op, me, kind, par = nodes[k]
            if kind == "client":
                if len(children[k]) != 1:
                    raise ValueError(f"{path}: client span with {len(children[k])} children (spans.py:33)")
                outs.setdefault(me, _Rows()).add(start, dur, tid, sid, nodes[children[k][0]][5])   # GetChildProcess
            elif kind == "server":
                other = "client_" + op if par < 0 else nodes[par][5]                      # GetParentProcess
                caller = (nodes[par][0], nodes[par][1]) if par >= 0 and nodes[par][6] == "client" else None
                ins.setdefault(me, _Rows()).add(start, dur, tid, sid, other, caller)
            else:
                raise ValueError(f"{path}: span.kind {kind!r} (executor.py:819)")
            stack.extend(reversed(children[k]))
        cnt += 1
        if cnt > max_traces:
            break

    lists = []
    for process, o in outs.items():                                                      # executor.py:1080
        if not o.start or process not in ins:
            continue
        L = _service_lists(process, ins[process], o)
        if L is not None:
            lists.append(L)
    if engine is not None and lists:
        return _services_device(engine, lists)
    return [_finish_service(L, *_truth_and_order_host(L)) for L in lists]


def _partition(rows: _Rows):
    """PartitionSpansByEndPoint (executor.py:1100-1109): {ep: row indices sorted by (start, end)},
    eps in first-appearance order, ties in list order."""
    parts: Dict[str, List[int]] = {}
    for k, ep in enumerate(rows.other):
        parts.setdefault(ep, []).append(k)
    start = np.asarray(rows.start, np.int64)
    end = start + np.asarray(rows.dur, np.int64)
    for ep, idx in parts.items():
        a = np.asarray(idx)
        order = np.lexsort((end[a], start[a]))       # stable, primary key start, secondary end
        parts[ep] = a[order]
    return parts, start, end


def _service_lists(process, i_rows: _Rows, o_rows: _Rows):
    """Partitions of one service (executor.py:1100-1128): None when it has more than one incoming endpoint."""
    in_parts, i_start, i_end = _partition(i_rows)
    out_parts, o_start, o_end = _partition(o_rows)
    if len(in_parts) > 1:
        return None                                                                      # "SKIPPING THIS PROCESS", :1121
    in_ep, in_idx = next(iter(in_parts.items()))
    given = list(out_parts.keys())
    return dict(process=process, in_ep=in_ep, in_idx=in_idx, given=given, out_parts=out_parts,
                i_start=i_start, i_end=i_end, o_start=o_start, o_end=o_end, i_rows=i_rows, o_rows=o_rows,
                i_tid=np.asarray(i_rows.tid)[in_idx])


def _truth_and_order_host(L):
    """GetGroundTruth (utils.py:22-32) and FindOrder's pruning (executor.py:248-266) in NumPy: the truth
    [E, n] in the given callee order and, per callee a, the bit mask of callees b whose edge a -> b some
    trace violates (x.end > y.start)."""
    given, out_parts, o_rows = L["given"], L["out_parts"], L["o_rows"]
    n = len(L["in_idx"])
    truth_given = np.full((len(given), n), -1, np.int32)
    for g, ep in enumerate(given):
        first: Dict[str, int] = {}
        for pos, k in enumerate(out_parts[ep]):
            first.setdefault(o_rows.tid[k], pos)
        truth_given[g] = [first.get(t, -1) for t in L["i_tid"]]
    if (truth_given < 0).any():
        raise ValueError(f"{L['process']}: an in-span has no child at some callee (FindOrder would raise KeyError)")
    ts = np.stack([L["o_start"][out_parts[ep]][truth_given[g]] for g, ep in enumerate(given)])     # [E, n]
    te = np.stack([L["o_end"][out_parts[ep]][truth_given[g]] for g, ep in enumerate(given)])
    violated = [0] * len(given)
    for a in range(len(given)):
        for b in range(len(given)):
            if a != b and bool((te[a] > ts[b]).any()):
                violated[a] |= 1 << b
    return truth_given, violated


def _finish_service(L, truth_given, violated) -> ServiceProblem:
    """FindOrder's graph (complete digraph minus the violated edges, executor.py:214-285), the
    topological callee order (traceweaver_v1.py:37-39) and the index-only problem."""
    import networkx as nx
    given, out_parts = L["given"], L["out_parts"]
    G = nx.DiGraph()
    for ep in given:
        G.add_node(ep)
    for a in given:
        for b in given:
            if a != b:
                G.add_edge(a, b)
    for a in range(len(given)):
        for b in range(len(given)):
            if a != b and (violated[a] >> b & 1) and G.has_edge(given[a], given[b]):
                G.remove_edge(given[a], given[b])                                        # x.end > y.start (:250, :262)
    topo = list(nx.topological_sort(G))                                                  # traceweaver_v1.py:37-39
    pos = {ep: e for e, ep in enumerate(topo)}
    g_of = [given.index(ep) for ep in topo]
    preds = [[pos[b] for b, _ in G.in_edges(ep)] for ep in topo]
    out_idx = [out_parts[ep] for ep in topo]
    i_rows, o_rows, in_idx = L["i_rows"], L["o_rows"], L["in_idx"]
    prob = Problem(in_start=L["i_start"][in_idx], in_end=L["i_end"][in_idx],
                   out_start=[L["o_start"][ix] for ix in out_idx], out_end=[L["o_end"][ix] for ix in out_idx],
                   preds=preds, name=L["process"])
    return ServiceProblem(
        name=L["process"], in_ep=L["in_ep"], out_eps_given=given, out_eps=topo, problem=prob,
        in_ids=[(i_rows.tid[k], i_rows.sid[k]) for k in in_idx],
        out_ids=[[(o_rows.tid[k], o_rows.sid[k]) for k in ix] for ix in out_idx],
        truth=np.ascontiguousarray(np.asarray(truth_given)[g_of]), graph_edges=list(G.edges()),
        in_caller_ids=[i_rows.caller[k] for k in in_idx])


def _service_problem(process, i_rows: _Rows, o_rows: _Rows) -> Optional[ServiceProblem]:
    L = _service_lists(process, i_rows, o_rows)
    if L is None:
        return None
    truth_given, violated = _truth_and_order_host(L)
    return _finish_service(L, truth_given, violated)


def _services_device(engine, lists) -> List[ServiceProblem]:
    """Ground truth and FindOrder of all services in ONE batch on the device (tw_ground_truth,
    tw_find_order: joins on the densely numbered trace id, csrc/tw_truth.cu); the per-service graphs
    (a handful of nodes) are then built on the host as before."""
    from . import truth as dev_truth
    number: Dict[str, int] = {}
    in_tr, out_tr, probs = [], [], []
    for L in lists:
        in_tr.append(np.fromiter((number.setdefault(t, len(number)) for t in L["i_tid"]), np.int32, len(L["i_tid"])))
        o_tid = L["o_rows"].tid
        out_tr.append([np.fromiter((number.setdefault(o_tid[k], len(number)) for k in L["out_parts"][ep]), np.int32,
                                   len(L["out_parts"][ep])) for ep in L["given"]])
        probs.append(dict(in_start=L["i_start"][L["in_idx"]], in_end=L["i_end"][L["in_idx"]],
                          out_start=[L["o_start"][L["out_parts"][ep]] for ep in L["given"]],
                          out_end=[L["o_end"][L["out_parts"][ep]] for ep in L["given"]]))
    tl = dev_truth.TraceLists(probs, in_tr, out_tr, len(number))
    truth = dev_truth.ground_truth(engine, tl)
    violated = dev_truth.find_order(engine, tl, truth)
    truth = truth.cpu().numpy()
    out = []
    for p, L in enumerate(lists):
        E, n = len(L["given"]), len(L["in_idx"])
        t0 = int(tl.arrays["prob_tuple_off"][p])
        e0 = int(tl.arrays["prob_ep_off"][p])
        out.append(_finish_service(L, truth[t0:t0 + E * n].reshape(E, n), [int(v) for v in violated[e0:e0 + E]]))
    return out


def to_host_batch(services: Sequence[ServiceProblem], skipped: list = None):
    """One bindable batch of the services that are in the accelerated regime (every callee list as
    long as the incoming list, i.e. no skip budget, traceweaver_v3.py:1138-1158).  Services outside it
    are left out — one of them would make tw_engine_bind reject the whole batch — and appended to
    `skipped` when the caller passes a list; the order of the others is kept.  Returns None when no
    service qualifies."""
    keep = []
    for s in services:
        if s.problem.in_accelerated_regime():
            keep.append(s)
        elif skipped is not None:
            skipped.append(s)
    return build_batch([s.problem for s in keep]) if keep else None


def accuracy(service: ServiceProblem, assign: np.ndarray) -> float:
    """utils.AccuracyForService (utils.py:34-60) on index arrays: fraction of in-spans whose child
    is right at EVERY callee.  `assign` is the engine's [E, n] block of this service."""
    ok = (np.asarray(assign).reshape(service.truth.shape) == service.truth).all(axis=0)
    return float(ok.mean()) if ok.size else 0.0


# ---------------------------------------------------------------------------------------------
# Accuracy on index arrays (helpers/utils.py:34-145), per service and per trace.  `truth`, `assign`
# are int32 [E, n]; `topk_idx` is [n, K, E] with `topk_cnt[i]` valid ranks; `in_trace[i]` the trace id.
# ---------------------------------------------------------------------------------------------
def topk_accuracy(truth: np.ndarray, topk_idx: np.ndarray, topk_cnt: np.ndarray) -> float:
    """utils.TopKAccuracyForService: an in-span counts when SOME rank matches the truth at every callee."""
    truth = np.asarray(truth)
    hit = (np.asarray(topk_idx) == truth.T[:, None, :]).all(axis=2)              # [n, K]
    valid = np.arange(hit.shape[1])[None, :] < np.asarray(topk_cnt)[:, None]
    ok = (hit & valid).any(axis=1)
    return float(ok.mean()) if ok.size else 0.0


def end_to_end_accuracy(in_traces: Sequence[Sequence[str]], truths: Sequence[np.ndarray],
                        assigns: Sequence[np.ndarray]) -> float:
    """utils.AccuracyEndToEnd over the solved services: a trace is right when every in-span it has
    in any of them got all its children right."""
    acc: Dict[str, bool] = {}
    for tids, truth, assign in zip(in_traces, truths, assigns):
        ok = (np.asarray(assign).reshape(np.asarray(truth).shape) == truth).all(axis=0)
        for t, good in zip(tids, ok):
            acc[t] = acc.get(t, True) and bool(good)
    return sum(acc.values()) / len(acc) if acc else 0.0


def end_to_end_topk_accuracy(in_traces: Sequence[Sequence[str]], truths: Sequence[np.ndarray],
                             topk_idxs: Sequence[np.ndarray], topk_cnts: Sequence[np.ndarray]) -> float:
    """utils.TopKAccuracyEndToEnd, with its order dependence: services in the given order; in the first
    service an in-span sets its trace's flag (the last in-span of the trace wins), in later services an
    in-span only touches traces that are still right."""
    acc: Dict[str, bool] = {}
    for s, (tids, truth, idx, cnt) in enumerate(zip(in_traces, truths, topk_idxs, topk_cnts)):
        truth = np.asarray(truth)
        hit = (np.asarray(idx) == truth.T[:, None, :]).all(axis=2)
        valid = np.arange(hit.shape[1])[None, :] < np.asarray(cnt)[:, None]
        ok = (hit & valid).any(axis=1)
        for t, good in zip(tids, ok):
            if s != 0 and acc[t] is False:
                continue
            acc[t] = bool(good)
    return sum(acc.values()) / len(acc) if acc else 0.0
