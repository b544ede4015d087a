"""End-to-end request trees of a solved batch (ConstructEndToEndTraces, helpers/utils.py:216, called from
executor.py:1210-1230): a thin wrapper around tw_assemble_traces (csrc/tw_traces.cu) plus its plain
restatement on the host.

Nodes: in-span g of the batch (global index, to_host_batch order) is node g, out-span j is node
n_in + j.  An out-span's parent is the in-span the assignment gave it to (predicted); an in-span's parent
is the client span of its RPC, `in_caller[g]` (observed: `caller_links`), -1 when that span is not in the
batch.  A node without a parent is a root: an in-span root is a reconstructed request, an out-span root a
detached fragment.  root[x] is -1 for a node on or under a cycle of links, size[r] counts the nodes of root
r.  Trace ids are never read here; they enter only `exact_requests`, the comparison with the truth."""
import ctypes as C
from typing import Sequence

import numpy as np
import torch

from . import _abi, _lib
from .batch import SPAN_ARRAYS, batch_struct
from .engine import _p, _to_device

_OFFSETS = ("prob_in_off", "prob_ep_off", "prob_tuple_off", "ep_out_off")


def node_count(hb):
    return int(hb.prob_in_off[-1]) + int(hb.ep_out_off[-1])


def caller_links(services: Sequence, hb) -> np.ndarray:
    """int32 [n_in]: the node id of every in-span's caller (ServiceProblem.in_caller_ids) in the batch
    to_host_batch(services) built, -1 for a request entering the batch or a caller outside it."""
    keep = [s for s in services if s.problem.in_accelerated_regime()]          # to_host_batch's selection
    n_in = int(hb.prob_in_off[-1])
    if hb.n_problems != len(keep) or sum(s.problem.n_in for s in keep) != n_in:
        raise ValueError("caller_links: `hb` is not to_host_batch(services)")
    node = {}
    for p, s in enumerate(keep):
        ep0 = int(hb.prob_ep_off[p])
        for e, ids in enumerate(s.out_ids):
            base = n_in + int(hb.ep_out_off[ep0 + e])
            for j, sid in enumerate(ids):
                node[sid] = base + j
    out = np.full(n_in, -1, np.int32)
    for p, s in enumerate(keep):
        i0 = int(hb.prob_in_off[p])
        for i, cid in enumerate(s.in_caller_ids):
            if cid is not None:
                out[i0 + i] = node.get(cid, -1)
    return out


def assemble(engine, hb, assign, in_caller):
    """tw_assemble_traces on the batch `hb` (host offsets; it need not be bound, a bound batch is not
    touched).  assign: the tw_pass_out.assign layout, in_caller: int32 [n_in]; device tensors or host
    arrays.  Returns device int32 tensors parent, root, size [n_nodes]."""
    dev = engine.device
    d = _to_device({k: hb.arrays[k] for k in _OFFSETS}, dev)
    links = {}
    for name, a in (("assign", assign), ("in_caller", in_caller)):
        links[name] = a if isinstance(a, torch.Tensor) else _to_device({name: np.asarray(a, np.int32).reshape(-1)},
                                                                        dev)[name]
    n_tuple, n_in = int(hb.prob_tuple_off[-1]), int(hb.prob_in_off[-1])
    if links["assign"].numel() != n_tuple or links["in_caller"].numel() != n_in:
        raise ValueError(f"assemble: assign must have {n_tuple} entries and in_caller {n_in}")
    view = _OffsetView(hb)
    dev_s = batch_struct(view, lambda k: d[k].data_ptr())
    host_s = batch_struct(view, lambda k: hb.arrays[k].ctypes.data)
    n = node_count(hb)
    out = {k: torch.empty(n, dtype=torch.int32, device=dev) for k in ("parent", "root", "size")}
    _lib.check(engine.lib.tw_assemble_traces(engine.h, C.byref(dev_s), C.byref(host_s), _p(links["assign"]),
                                             _p(links["in_caller"]), _p(out["parent"]), _p(out["root"]),
                                             _p(out["size"]), engine.stream), "tw_assemble_traces")
    return out


class _OffsetView:
    """The offset tables of a batch, without its span arrays or term tables: all tw_assemble_traces reads."""

    def __init__(self, hb):
        self.arrays = {k: hb.arrays[k] for k in _OFFSETS}
        self.n_problems = hb.n_problems


def exact_requests(root_pred: torch.Tensor, root_true: torch.Tensor, n_in: int) -> torch.Tensor:
    """int8 [n_in] on the device: for an in-span root r of the prediction 1 iff its request is exact (the
    nodes with root r are the same under both joins), else 0; -1 for an in-span that is not a root.
    A node whose roots differ spoils both of them: one mismatch test and two scatters."""
    n = root_pred.numel()
    bad = torch.zeros(n + 1, dtype=torch.bool, device=root_pred.device)
    mis = root_pred != root_true
    for r in (root_pred[mis], root_true[mis]):
        bad[torch.where(r >= 0, r, n).long()] = True                  # -1 (a cycle) lands in the spare slot
    node = torch.arange(n_in, dtype=root_pred.dtype, device=root_pred.device)
    is_root = root_pred[:n_in] == node
    return torch.where(is_root, (~bad[:n_in]).to(torch.int8), torch.full_like(is_root, -1, dtype=torch.int8))


# ---------------------------------------------------------------------------------------------
# Host restatement: the same arrays by walking each node up to its root (the reference the tests compare
# tw_assemble_traces with; no GPU needed).
# ---------------------------------------------------------------------------------------------
def _smallest_repeat(x):
    v, c = np.unique(x, return_counts=True)
    return int(v[c > 1][0]) if (c > 1).any() else None


def parents_host(hb, assign, in_caller) -> np.ndarray:
    """int64 [n_nodes]: the parent of every node, or -1; ValueError naming the smallest malformed node."""
    n_in, n_out = int(hb.prob_in_off[-1]), int(hb.ep_out_off[-1])
    assign = np.asarray(assign, np.int64).reshape(-1)
    c = np.asarray(in_caller, np.int64).reshape(-1)
    parent = np.full(n_in + n_out, -1, np.int64)
    wrong = np.flatnonzero((c != -1) & ((c < n_in) | (c >= n_in + n_out)))
    if wrong.size:
        raise ValueError(f"in-span node {wrong[0]} has a caller that is not an out-span node")
    twice = _smallest_repeat(c[c >= 0])
    if twice is not None:
        raise ValueError(f"out-span node {twice} is the caller of two in-spans")
    parent[:n_in] = c
    # tuple g = (service p, callee e, in-span i), g = tuple_off[p] + e * n_p + i
    off = np.asarray(hb.prob_tuple_off, np.int64)
    p = np.repeat(np.arange(hb.n_problems), np.diff(off))
    n_p = np.diff(np.asarray(hb.prob_in_off, np.int64))[p]
    local = np.arange(off[-1]) - off[p]
    ep = np.asarray(hb.prob_ep_off, np.int64)[p] + local // n_p
    node_in = np.asarray(hb.prob_in_off, np.int64)[p] + local % n_p
    out_off = np.asarray(hb.ep_out_off, np.int64)
    has = assign >= 0
    outside = np.flatnonzero(has & (assign >= out_off[ep + 1] - out_off[ep]))
    if outside.size:
        raise ValueError(f"in-span node {node_in[outside].min()} has a child index outside its callee's list")
    x = n_in + out_off[ep[has]] + assign[has]
    twice = _smallest_repeat(x)
    if twice is not None:
        raise ValueError(f"out-span node {twice} is the child of two in-spans")
    parent[x] = node_in[has]
    return parent


def assemble_host(hb, assign, in_caller, vector_steps=64):
    """parent, root, size (int32 numpy [n_nodes]) as tw_assemble_traces computes them; ValueError where it
    returns TW_ERR_INVALID.  Every node climbs its links one at a time: `vector_steps` steps for all nodes
    at once, then node by node for what is left (deeper trees and cycles)."""
    parent = parents_host(hb, assign, in_caller)
    n = parent.shape[0]
    top = np.arange(n)
    for _ in range(vector_steps):
        up = parent[top]
        if not (up >= 0).any():
            break
        top = np.where(up >= 0, up, top)
    root = np.where(parent[top] < 0, top, -2)        # -2: not reached yet
    on_path = np.zeros(n, bool)
    for x in np.flatnonzero(root == -2):
        path, y = [], int(x)
        while True:
            if root[y] != -2:
                r = int(root[y])
                break
            if on_path[y]:                           # back on its own path: y lies on a cycle
                r = -1
                break
            on_path[y] = True
            path.append(y)
            if parent[y] < 0:
                r = y
                break
            y = int(parent[y])
        root[path] = r
        on_path[path] = False
    size = np.bincount(root[root >= 0], minlength=n)
    return parent.astype(np.int32), root.astype(np.int32), size.astype(np.int32)


# ---------------------------------------------------------------------------------------------
# Critical paths (tw_critical_paths, csrc/tw_critical_path.cu): where each request's time went.  This is the
# project's own definition; the reference's consumers of its traces are not part of it.  A request is an
# in-span root r; its window is [start_r, max(start_r, end_r)] and its latency the window's length.  Windows
# are handed down the tree, and every node that gets one is on the path.  Its self time is the part of its
# window it hands to no child:
#   in-span with window [a, b]: every child out-span is clipped to [a, b] and is eligible iff what is left,
#     [s_k, e_k], is not empty.  With c = b: among the unchosen eligible children with s_k < c, the one with
#     the largest min(e_k, c) (the lowest callee position on a tie) gets [s_k, min(e_k, c)]; c - min(e_k, c)
#     is self time, and c becomes s_k.  When no child qualifies, c - a is self time.  So sequential calls
#     are all on the path; of parallel calls the one that ends last is, with any call still running when it
#     started (truncated); a call nested in a chosen one is not.
#   out-span with window [a, b]: its child in-span (the one whose caller it is) is on the path iff its
#     interval clipped to [a, b] is not empty, and gets that window; the rest of [a, b] is self time:
#     network and queueing, or the whole callee when its server span is not in the batch.
# The self times of a request's on-path nodes add up to its latency (exactly for int64 times).  The culprit
# of a request is its on-path node with the largest self time, the smallest node id on a tie.
# ---------------------------------------------------------------------------------------------
_CP_KEYS = ("root", "on_path", "self_us", "culprit", "server_us", "server_visits", "call_us", "requests")


def upload_spans(engine, hb):
    """The four span arrays of `hb` on the device (int64, or float64 for a time-compressed batch)."""
    return _to_device({k: hb.arrays[k] for k in SPAN_ARRAYS}, engine.device)


class _SpanView(_OffsetView):
    """The offset tables and span arrays of a batch: all tw_critical_paths reads."""

    def __init__(self, hb, spans):
        super().__init__(hb)
        self.arrays.update(spans)


def critical_paths(engine, hb, assign, in_caller, slow_us, spans=None):
    """tw_critical_paths on the batch `hb` (host offsets; it need not be bound, a bound batch is not
    touched).  assign, in_caller as for assemble; slow_us: requests with latency >= slow_us form the second
    column of the sums; spans: upload_spans(engine, hb) when the caller already has it.  Returns device
    tensors: root int32 [N], on_path uint8 [N], self_us float64 [N], culprit int32 [n_in], server_us float64
    [P, 2], server_visits int32 [P, 2], call_us float64 [n_ep, 2], requests int32 [2].  Trees of any depth
    are walked, with the same results whatever the number of level launches."""
    dev = engine.device
    d = _to_device({k: hb.arrays[k] for k in _OFFSETS}, dev)
    d.update(spans if spans is not None else upload_spans(engine, hb))
    links = {}
    for name, a in (("assign", assign), ("in_caller", in_caller)):
        links[name] = a if isinstance(a, torch.Tensor) else _to_device({name: np.asarray(a, np.int32).reshape(-1)},
                                                                        dev)[name]
    n_tuple, n_in = int(hb.prob_tuple_off[-1]), int(hb.prob_in_off[-1])
    if links["assign"].numel() != n_tuple or links["in_caller"].numel() != n_in:
        raise ValueError(f"critical_paths: assign must have {n_tuple} entries and in_caller {n_in}")
    view = _SpanView(hb, {k: d[k] for k in SPAN_ARRAYS})
    dev_s = batch_struct(view, lambda k: d[k].data_ptr())
    host_s = batch_struct(_OffsetView(hb), lambda k: hb.arrays[k].ctypes.data)
    f64 = _abi.fill(_abi.TwTimesF64, d) if d["in_start"].dtype == torch.float64 else None
    n, P, n_ep = node_count(hb), hb.n_problems, int(hb.prob_ep_off[-1])
    out = dict(root=torch.empty(n, dtype=torch.int32, device=dev), on_path=torch.empty(n, dtype=torch.uint8, device=dev),
               self_us=torch.empty(n, dtype=torch.float64, device=dev),
               culprit=torch.empty(n_in, dtype=torch.int32, device=dev),
               server_us=torch.empty((P, 2), dtype=torch.float64, device=dev),
               server_visits=torch.empty((P, 2), dtype=torch.int32, device=dev),
               call_us=torch.empty((n_ep, 2), dtype=torch.float64, device=dev),
               requests=torch.empty(2, dtype=torch.int32, device=dev))
    o = _abi.fill(_abi.TwCriticalOut, out)
    _lib.check(engine.lib.tw_critical_paths(engine.h, C.byref(dev_s), C.byref(host_s),
                                            C.byref(f64) if f64 is not None else None, _p(links["assign"]),
                                            _p(links["in_caller"]), C.c_double(slow_us), C.byref(o),
                                            engine.stream), "tw_critical_paths")
    return out


def request_latencies(spans, in_caller):
    """Device tensors: the request roots (in-spans without a caller: the in-span roots of the join) and
    their latencies, float64 microseconds, as tw_critical_paths forms them."""
    req = torch.nonzero(in_caller == -1).reshape(-1)
    a, e = spans["in_start"][req], spans["in_end"][req]
    return req.to(torch.int32), (torch.maximum(a, e) - a).to(torch.float64)


def lower_quantile(x: torch.Tensor, q: float) -> float:
    """The lower q-quantile of x (torch.quantile's "lower" interpolation, for any size): an element of x;
    +inf for an empty x."""
    if x.numel() == 0:
        return float("inf")
    k = int(np.floor(q * (x.numel() - 1)))
    return float(torch.sort(x).values[k])


def critical_paths_host(hb, assign, in_caller, slow_us):
    """The arrays of critical_paths (numpy), by walking every request from its root as defined above;
    ValueError where tw_critical_paths returns TW_ERR_INVALID.  Also latency [n_requests] (float64) of the
    requests in node order."""
    _, root, _ = assemble_host(hb, assign, in_caller)
    n_in, n_out = int(hb.prob_in_off[-1]), int(hb.ep_out_off[-1])
    n, P, n_ep = n_in + n_out, hb.n_problems, int(hb.prob_ep_off[-1])
    f64 = hb.float_times
    zero = 0.0 if f64 else 0
    in_s, in_e = hb.in_start.tolist(), hb.in_end.tolist()
    out_s, out_e = hb.out_start.tolist(), hb.out_end.tolist()
    # the child out-span of every in-span per callee position (-1: none), and every out-span's child in-span
    assign = np.asarray(assign, np.int64).reshape(-1)
    off = np.asarray(hb.prob_tuple_off, np.int64)
    p = np.repeat(np.arange(P), np.diff(off))
    n_p = np.diff(np.asarray(hb.prob_in_off, np.int64))[p]
    local = np.arange(off[-1]) - off[p]
    pos = local // n_p
    ep = np.asarray(hb.prob_ep_off, np.int64)[p] + pos
    node_in = np.asarray(hb.prob_in_off, np.int64)[p] + local % n_p
    kids = np.full((n_in, 8), -1, np.int64)
    has = assign >= 0
    kids[node_in[has], pos[has]] = np.asarray(hb.ep_out_off, np.int64)[ep[has]] + assign[has]
    n_callee = np.diff(np.asarray(hb.prob_ep_off, np.int64))[np.repeat(np.arange(P), np.diff(hb.prob_in_off))]
    kids = [row[:E] for row, E in zip(kids.tolist(), n_callee.tolist())]
    c = np.asarray(in_caller, np.int64).reshape(-1)
    callee_in = np.full(n_out, -1, np.int64)
    callee_in[c[c >= 0] - n_in] = np.flatnonzero(c >= 0)
    callee_in = callee_in.tolist()

    on_path = np.zeros(n, np.uint8)
    self_us = np.zeros(n, np.float64)
    culprit = np.full(n_in, -1, np.int32)
    slow = np.zeros(n, bool)
    requests = [r for r in range(n_in) if root[r] == r]
    latency = np.zeros(len(requests), np.float64)
    for q, r in enumerate(requests):
        a0 = in_s[r]
        b0 = max(in_e[r], a0)
        latency[q] = float(b0 - a0)
        todo = [(r, a0, b0)]                          # in-spans on the path with their windows
        nodes = []
        while todo:
            x, a, b = todo.pop()
            nodes.append(x)
            cand = []                                 # eligible children in callee order: [start, end, out-span]
            for k in kids[x]:
                if k >= 0:
                    s, e = max(out_s[k], a), min(out_e[k], b)
                    if e > s:
                        cand.append((s, e, k))
            cur, own, chosen = b, zero, set()
            while True:
                best = None
                for idx, (s, e, k) in enumerate(cand):
                    if idx in chosen or not s < cur:
                        continue
                    if best is None or min(e, cur) > best[1]:
                        best = (idx, min(e, cur))
                if best is None:
                    break
                idx, end = best
                chosen.add(idx)
                s, _, k = cand[idx]
                own = own + (cur - end)
                cur = s
                # the out-span k with window [s, end] and its child in-span
                node = n_in + k
                nodes.append(node)
                y = callee_in[k]
                rest = end - s
                if y >= 0:
                    lo, hi = max(in_s[y], s), min(in_e[y], end)
                    if hi > lo:
                        rest = (end - s) - (hi - lo)
                        todo.append((y, lo, hi))
                self_us[node] = float(rest)
            self_us[x] = float(own + (cur - a))
        on_path[nodes] = 1
        slow[nodes] = latency[q] >= slow_us
        best = max(nodes, key=lambda v: (self_us[v], -v))
        culprit[r] = best
    server_us = np.zeros((P, 2))
    server_visits = np.zeros((P, 2), np.int32)
    call_us = np.zeros((n_ep, 2))
    in_prob = np.repeat(np.arange(P), np.diff(hb.prob_in_off))
    out_ep = np.repeat(np.arange(n_ep), np.diff(hb.ep_out_off))
    for col, mask in enumerate((on_path == 1, (on_path == 1) & slow)):
        server_us[:, col] = np.bincount(in_prob, weights=np.where(mask[:n_in], self_us[:n_in], 0.0), minlength=P)
        server_visits[:, col] = np.bincount(in_prob, weights=mask[:n_in], minlength=P).astype(np.int32)
        call_us[:, col] = np.bincount(out_ep, weights=np.where(mask[n_in:], self_us[n_in:], 0.0), minlength=n_ep)
    return dict(root=root, on_path=on_path, self_us=self_us, culprit=culprit, server_us=server_us,
                server_visits=server_visits, call_us=call_us,
                requests=np.array([len(requests), int((latency >= slow_us).sum())], np.int32), latency=latency)
