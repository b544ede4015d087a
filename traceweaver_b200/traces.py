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
from types import SimpleNamespace
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


def upload_inputs(engine, hb, who, **arrays):
    """The input arrays of the request-tree entry points on the engine's device, by name: assign, in_caller,
    score, code, topk_score, topk_idx, topk_cnt (device tensors or host arrays), each flat and contiguous in
    the dtype the kernels read.  ValueError naming the wrapper `who` and the array when its size does not fit
    the batch `hb`."""
    n_tuple, n_in, K = int(hb.prob_tuple_off[-1]), int(hb.prob_in_off[-1]), _abi.TW_K
    want = dict(assign=(n_tuple, np.int32, torch.int32), in_caller=(n_in, np.int32, torch.int32),
                score=(n_in, np.float64, torch.float64), code=(n_in, np.uint8, torch.uint8),
                topk_score=(K * n_in, np.float64, torch.float64), topk_idx=(K * n_tuple, np.int32, torch.int32),
                topk_cnt=(n_in, np.uint8, torch.uint8))
    dev = engine.device
    d = {}
    for name, a in arrays.items():
        size, npt, tt = want[name]
        if isinstance(a, torch.Tensor):
            t = a.to(device=dev, dtype=tt).contiguous().reshape(-1)
        else:
            t = _to_device({name: np.ascontiguousarray(np.asarray(a, npt).reshape(-1))}, dev)[name]
        if t.numel() != size:
            raise ValueError(f"{who}: {name} must have {size} entries for this batch, not {t.numel()}")
        d[name] = t
    return d


def _batch_structs(engine, hb, spans=None):
    """The TwBatch of `hb`'s offset tables on the device and on the host, the device one also pointing at
    `spans` (upload_spans) when given: all the request-tree entry points read of a batch.  Also the device
    tensors, which must outlive the call."""
    view = SimpleNamespace(n_problems=hb.n_problems, arrays={k: hb.arrays[k] for k in _OFFSETS})
    d = _to_device(view.arrays, engine.device)
    host_s = batch_struct(view, lambda k: hb.arrays[k].ctypes.data)
    if spans is not None:
        d.update(spans)
        view.arrays.update(spans)
    return batch_struct(view, lambda k: d[k].data_ptr()), host_s, d


def assemble(engine, hb, assign, in_caller):
    """tw_assemble_traces on the batch `hb` (host offsets; it need not be bound, a bound batch is not
    touched).  assign: the tw_pass_out.assign layout, in_caller: int32 [n_in]; device tensors or host
    arrays.  Returns device int32 tensors parent, root, size [n_nodes]."""
    links = upload_inputs(engine, hb, "assemble", assign=assign, in_caller=in_caller)
    dev_s, host_s, _keep = _batch_structs(engine, hb)
    n = node_count(hb)
    out = {k: torch.empty(n, dtype=torch.int32, device=engine.device) for k in ("parent", "root", "size")}
    _lib.check(engine.lib.tw_assemble_traces(engine.h, C.byref(dev_s), C.byref(host_s), _p(links["assign"]),
                                             _p(links["in_caller"]), _p(out["parent"]), _p(out["root"]),
                                             _p(out["size"]), engine.stream), "tw_assemble_traces")
    return out


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
def _tuples(hb):
    """Every tuple g = tuple_off[p] + e * n_p + i of the batch (service p, callee position e, in-span i) as
    its global callee ep, its callee position e and its in-span node: three int64 arrays [n_tuple]."""
    off = np.asarray(hb.prob_tuple_off, np.int64)
    p = np.repeat(np.arange(hb.n_problems), np.diff(off))
    n_p = np.diff(np.asarray(hb.prob_in_off, np.int64))[p]
    local = np.arange(off[-1]) - off[p]
    pos = local // n_p
    return np.asarray(hb.prob_ep_off, np.int64)[p] + pos, pos, np.asarray(hb.prob_in_off, np.int64)[p] + local % n_p


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
    ep, _, node_in = _tuples(hb)
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


def critical_paths(engine, hb, assign, in_caller, slow_us, spans=None):
    """tw_critical_paths on the batch `hb` (host offsets; it need not be bound, a bound batch is not
    touched).  assign, in_caller as for assemble; slow_us: requests with latency >= slow_us form the second
    column of the sums; spans: upload_spans(engine, hb) when the caller already has it.  Returns device
    tensors: root int32 [N], on_path uint8 [N], self_us float64 [N], culprit int32 [n_in], server_us float64
    [P, 2], server_visits int32 [P, 2], call_us float64 [n_ep, 2], requests int32 [2].  Trees of any depth
    are walked, with the same results whatever the number of level launches."""
    dev = engine.device
    links = upload_inputs(engine, hb, "critical_paths", assign=assign, in_caller=in_caller)
    spans = spans if spans is not None else upload_spans(engine, hb)
    dev_s, host_s, _keep = _batch_structs(engine, hb, spans)
    f64 = _abi.fill(_abi.TwTimesF64, spans) if spans["in_start"].dtype == torch.float64 else None
    n, n_in, P, n_ep = node_count(hb), int(hb.prob_in_off[-1]), hb.n_problems, int(hb.prob_ep_off[-1])
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
    ep, pos, node_in = _tuples(hb)
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


# ---------------------------------------------------------------------------------------------
# Request confidence (tw_request_confidence, csrc/tw_confidence.cu): how sure the reconstruction of each
# request is, without a ground truth.  This is the project's own definition.  Every in-span x is one
# reconstruction decision.  Its choice probability p_x is the chosen tuple's share of the likelihood among
# the alternatives the engine listed:
#   p_x = 0 unless code[x] == TW_ASSESS_SCORED (NA, out of range, infeasible; also when score[x] is -inf);
#   else, with A the listed ranks r < topk_cnt[x] of the final no-deletion top-K whose tuple differs from
#   the chosen one at some callee position, s_c = score[x] and m = max(s_c, max_A s_r):
#     S = exp(s_c - m) + sum over r in A, ascending, of exp(s_r - m),   p_x = exp(s_c - m) / S.
#   A single candidate gives 1; a chosen tuple the list does not hold counts with its own score.
#   ell_x = -log p_x, formed as log(S) + (m - s_c); +inf where p_x == 0 (also when exp underflows).
# It ignores the windows' conflicts and the tuples beyond rank K, so it is pessimistic: a ranking signal,
# not a calibrated probability, and not an accuracy.  Per request r (an in-span root of the join; in-spans
# on or under a cycle or in a detached fragment belong to none): decisions[r], zero[r] (decisions with
# p = 0), log_conf[r] = the sum of the others' ell, each rounded to a multiple of 2^-32 nats and added as
# int64; conf[r] = exp(-log_conf[r] * 2^-32), 0 when zero[r] > 0; weakest[r] the decision with the smallest
# p (smallest node id on a tie) and weakest_p[r] its p.  Per service est_accuracy = the mean p of its
# in-spans; per batch the request count and expected_exact = the sum of conf.  exp and log are the engine's
# own (conf_exp / conf_log below, the same operations as tw_core.cuh), so every float here is bit-identical
# to the device's; the sums follow the kernels' fixed order (_cta_sum).
# ---------------------------------------------------------------------------------------------
_CONF_KEYS = ("root", "p", "ell", "decisions", "zero", "log_conf", "conf", "weakest", "weakest_p", "est_accuracy",
              "requests", "expected_exact")
_LN2_HI, _LN2_LO, _RINT = 0.6931471803691238, 1.9082149292705877e-10, 6755399441055744.0
_EXP_C = (1.6059043836821613e-10, 2.08767569878681e-09, 2.505210838544172e-08, 2.755731922398589e-07,
          2.7557319223985893e-06, 2.48015873015873e-05, 0.0001984126984126984, 0.001388888888888889,
          0.008333333333333333, 0.041666666666666664, 0.16666666666666666, 0.5, 1.0, 1.0)
_LOG_C = (0.047619047619047616, 0.05263157894736842, 0.058823529411764705, 0.06666666666666667,
          0.07692307692307693, 0.09090909090909091, 0.1111111111111111, 0.14285714285714285, 0.2,
          0.3333333333333333)


def conf_exp(d):
    """exp(d) for d <= 0 as tw_core.cuh's conf_exp computes it (0 below -746 and for NaN), elementwise."""
    d = np.asarray(d, np.float64)
    ok = d >= -746.0
    x = np.where(ok, d, 0.0)
    nf = (x * 1.4426950408889634 + _RINT) - _RINT
    r = (x - nf * _LN2_HI) - nf * _LN2_LO
    q = np.full_like(x, _EXP_C[0])
    for c in _EXP_C[1:]:
        q = q * r + c
    n = nf.astype(np.int64)
    n1 = n >> 1
    pow2 = lambda k: ((k + 1023) << 52).astype(np.int64).view(np.float64)
    return np.where(ok, (q * pow2(n1)) * pow2(n - n1), 0.0)


def conf_log(x):
    """log(x) for positive normal x as tw_core.cuh's conf_log computes it, elementwise."""
    u = np.asarray(x, np.float64).view(np.int64)
    k = (u >> 52) - 1023
    f = ((u & 0x000fffffffffffff) | 0x3ff0000000000000).view(np.float64)
    big = f > 1.4142135623730951
    f = np.where(big, f * 0.5, f)
    k = k + big
    s = (f - 1.0) / (f + 1.0)
    z = s * s
    q = np.full_like(s, _LOG_C[0])
    for c in _LOG_C[1:]:
        q = q * z + c
    s2 = s + s
    kf = k.astype(np.float64)
    return kf * _LN2_HI + (kf * _LN2_LO + (s2 + (s2 * z) * q))


def _cta_sum(v):
    """The kernels' fixed-order sum of v (one CTA of 256 threads: thread t adds v[t], v[t + 256], ... in order,
    a butterfly per warp of 32, then the warps in order)."""
    v = np.asarray(v, np.float64)
    lanes = np.zeros(256)
    for lo in range(0, len(v), 256):
        row = v[lo:lo + 256]
        lanes[:len(row)] = lanes[:len(row)] + row
    w = lanes.reshape(8, 32)
    for d in (16, 8, 4, 2, 1):
        w = w + w[:, np.arange(32) ^ d]
    s = w[0, 0]
    for k in range(1, 8):
        s = s + w[k, 0]
    return float(s)


def _topk_arrays(topk, n_in, n_tuple):
    sc = np.asarray(topk["topk_score"], np.float64).reshape(-1)
    idx = np.asarray(topk["topk_idx"], np.int32).reshape(-1)
    cnt = np.asarray(topk["topk_cnt"], np.uint8).reshape(-1)
    if sc.size != _abi.TW_K * n_in or idx.size != _abi.TW_K * n_tuple or cnt.size != n_in:
        raise ValueError(f"request_confidence: topk_score must have {_abi.TW_K * n_in} entries, topk_idx "
                         f"{_abi.TW_K * n_tuple} and topk_cnt {n_in}")
    return sc, idx, cnt


def request_confidence(engine, hb, assign, in_caller, score, code, topk):
    """tw_request_confidence on the batch `hb` (host offsets; it need not be bound, a bound batch is not
    touched).  assign, in_caller as for assemble; score float64 / code uint8 [n_in] of the chosen tuples
    (tw_score_assignments: solve(want_likelihood=True)'s chosen_score / chosen_code, or BatchSolver.score);
    topk: topk_score [n_in, K], topk_idx, topk_cnt of the final no-deletion top-K (solve(want_scores=True)).
    Device tensors or host arrays.  Returns device tensors: root int32 [N]; p, ell float64, decisions, zero
    int32, log_conf int64 (units of 2^-32 nats), conf float64, weakest int32, weakest_p float64 [n_in];
    est_accuracy float64 [P]; requests int32 [1]; expected_exact float64 [1].  Definition above."""
    dev = engine.device
    links = upload_inputs(engine, hb, "request_confidence", assign=assign, in_caller=in_caller, score=score,
                          code=code, topk_score=topk["topk_score"], topk_idx=topk["topk_idx"],
                          topk_cnt=topk["topk_cnt"])
    dev_s, host_s, _keep = _batch_structs(engine, hb)
    n, n_in, P = node_count(hb), int(hb.prob_in_off[-1]), hb.n_problems
    out = dict(root=torch.empty(n, dtype=torch.int32, device=dev))
    for k, dt in (("p", torch.float64), ("ell", torch.float64), ("decisions", torch.int32), ("zero", torch.int32),
                  ("log_conf", torch.int64), ("conf", torch.float64), ("weakest", torch.int32),
                  ("weakest_p", torch.float64)):
        out[k] = torch.empty(n_in, dtype=dt, device=dev)
    out.update(est_accuracy=torch.empty(P, dtype=torch.float64, device=dev),
               requests=torch.empty(1, dtype=torch.int32, device=dev),
               expected_exact=torch.empty(1, dtype=torch.float64, device=dev))
    top = _abi.fill(_abi.TwScoreOut, {k: links[k] for k in ("topk_score", "topk_idx", "topk_cnt")})
    o = _abi.fill(_abi.TwConfidenceOut, out)
    _lib.check(engine.lib.tw_request_confidence(engine.h, C.byref(dev_s), C.byref(host_s), _p(links["assign"]),
                                                _p(links["in_caller"]), _p(links["score"]), _p(links["code"]),
                                                C.byref(top), C.byref(o), engine.stream), "tw_request_confidence")
    return out


def choice_host(hb, assign, score, code, topk):
    """p, ell (float64 [n_in]) and the fixed-point ell (int64, -1 where p == 0) of every in-span, as defined
    above (vectorised over the in-spans of each service)."""
    n_in, n_tuple = int(hb.prob_in_off[-1]), int(hb.prob_tuple_off[-1])
    K = _abi.TW_K
    tks, tki, cnt = _topk_arrays(topk, n_in, n_tuple)
    tks = tks.reshape(n_in, K)
    assign = np.asarray(assign, np.int32).reshape(-1)
    score = np.asarray(score, np.float64).reshape(-1)
    code = np.asarray(code, np.uint8).reshape(-1)
    if assign.size != n_tuple or score.size != n_in or code.size != n_in:
        raise ValueError(f"request_confidence: assign must have {n_tuple} entries, score and code {n_in}")
    p_out = np.zeros(n_in)
    ell = np.full(n_in, np.inf)
    q = np.full(n_in, -1, np.int64)
    for pb in range(hb.n_problems):
        i0, i1 = int(hb.prob_in_off[pb]), int(hb.prob_in_off[pb + 1])
        n, E = i1 - i0, int(hb.prob_ep_off[pb + 1] - hb.prob_ep_off[pb])
        t0 = int(hb.prob_tuple_off[pb])
        chosen = assign[t0:t0 + n * E].reshape(E, n).T                       # [n, E]
        idx = tki[K * t0:K * (t0 + n * E)].reshape(n, K, E)
        c = np.minimum(cnt[i0:i1], K)
        s_c = score[i0:i1]
        live = (code[i0:i1] == _abi.TW_ASSESS_SCORED) & (s_c > -np.inf)
        alt = (idx != chosen[:, None, :]).any(axis=2) & (np.arange(K)[None, :] < c[:, None])
        s = tks[i0:i1]
        m = s_c.copy()
        for r in range(K):
            m = np.where(alt[:, r] & (s[:, r] > m), s[:, r], m)
        a = conf_exp(np.where(live, s_c - m, 0.0))
        S = a.copy()
        for r in range(K):
            S = np.where(alt[:, r], S + conf_exp(np.where(alt[:, r], s[:, r] - m, 0.0)), S)
        pp = np.where(live, a / np.where(live, S, 1.0), 0.0)
        pos = pp > 0.0
        lg = conf_log(np.where(pos, S, 1.0)) + np.where(pos, m - s_c, 0.0)
        p_out[i0:i1] = np.where(pos, pp, 0.0)
        ell[i0:i1] = np.where(pos, lg, np.inf)
        q[i0:i1] = np.where(pos, ((np.where(pos, lg, 0.0) * 4294967296.0 + _RINT) - _RINT).astype(np.int64), -1)
    return p_out, ell, q


def request_confidence_host(hb, assign, in_caller, score, code, topk):
    """The arrays of request_confidence (numpy) from the definition above, with the join of assemble_host;
    ValueError where tw_request_confidence returns TW_ERR_INVALID or TW_ERR_RANGE_LIMIT.  Also q, the
    fixed-point ell of every in-span (-1 where p == 0)."""
    _, root, _ = assemble_host(hb, assign, in_caller)
    n_in, P = int(hb.prob_in_off[-1]), hb.n_problems
    p, ell, q = choice_host(hb, assign, score, code, topk)
    r = root[:n_in].astype(np.int64)
    mine = (r >= 0) & (r < n_in)
    decisions = np.bincount(r[mine], minlength=n_in).astype(np.int32)
    zero = np.bincount(r[mine & (q < 0)], minlength=n_in).astype(np.int32)
    log_conf = np.zeros(n_in, np.int64)
    np.add.at(log_conf, r[mine & (q >= 0)], q[mine & (q >= 0)])
    big = np.flatnonzero(decisions >= 1 << 21)
    if big.size:
        raise ValueError(f"the request rooted at in-span node {big[0]} has 2^21 or more decisions")
    is_root = r == np.arange(n_in)
    conf = np.full(n_in, np.nan)
    conf[is_root] = np.where(zero[is_root] > 0, 0.0, conf_exp(log_conf[is_root].astype(np.float64) * -2.0 ** -32))
    weakest = np.full(n_in, -1, np.int32)
    weakest_p = np.full(n_in, np.nan)
    x = np.flatnonzero(mine)
    order = np.lexsort((x, p[x], r[x]))                   # by request, then p, then node id
    xs = x[order]
    first = np.ones(len(xs), bool)
    first[1:] = r[xs][1:] != r[xs][:-1]
    weakest[r[xs[first]]] = xs[first]
    weakest_p[r[xs[first]]] = p[xs[first]]
    est = np.array([_cta_sum(p[int(hb.prob_in_off[k]):int(hb.prob_in_off[k + 1])]) /
                    float(hb.prob_in_off[k + 1] - hb.prob_in_off[k]) for k in range(P)])
    seg_conf = [_cta_sum(np.where(is_root, conf, 0.0)[int(hb.prob_in_off[k]):int(hb.prob_in_off[k + 1])])
                for k in range(P)]
    return dict(root=root, p=p, ell=ell, decisions=decisions, zero=zero, log_conf=log_conf, conf=conf,
                weakest=weakest, weakest_p=weakest_p, est_accuracy=est,
                requests=np.array([int(is_root.sum())], np.int32), expected_exact=np.array([_cta_sum(seg_conf)]),
                q=q)
