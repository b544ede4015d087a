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

from . import _lib
from .batch import batch_struct
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
