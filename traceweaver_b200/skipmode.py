"""Skip / cache mode of the path (SURVEY.md §8 rows a11, a12, f-4): host mirror around `tw_skip_solve`.

A service some of whose outgoing lists do not hold one span per incoming span (cache hits of
exps/exp2: executor.py:1150-1152 -> helpers/transforms.py:153-238) takes ONE iteration with skip
spans in the reference (traceweaver_v3.py = V3: :1138-1158).  The search, scoring, stitching and the
parent search of BuildDistributions run on the device (csrc/tw_skip.cu).  What stays here is what the
reference computes with NumPy library calls whose tie behaviour is part of the result, and the state
its predictor instance carries from one service to the next:

  * the time windows (V3:973-985) — `self.time_windows` is never reset (V3:45), so the list keeps
    growing across services and FetchSkipFromWindow (V3:820-842) searches all of it;
  * WaterFill (V3:863-917): tie order among windows with equal span counts is `np.argsort`'s;
  * np.mean / np.std of the BuildDistributions samples (V3:171-172); `self.distribution_values`
    is never reset either (V3:40), so the sample lists accumulate per (endpoint, endpoint) key.
"""
import ctypes as C

import numpy as np
import torch

from . import _abi, _lib
from .batch import Problem, batch_struct, build_batch
from .engine import _p, _to_device

MAX_WINDOW = _abi.TW_MAX_WINDOW


class SkipState:
    """What a TraceWeaverV3 instance of the reference keeps between FindAssignments calls and the skip
    regime reads: `time_windows` [(start, end, expected)], `distribution_values` {(ep, ep): [samples]}."""

    def __init__(self):
        self.time_windows = []
        self.distribution_values = {}


def new_time_windows(in_start, in_end):
    """Windows of 30 incoming spans appended by TallySkipSpans, V3:973-985."""
    n = len(in_start)
    bounds = [int(in_end[i]) for i in range(MAX_WINDOW, n - 1, MAX_WINDOW)]
    edges = [int(in_start[0])] + bounds
    wins = [(edges[k], edges[k + 1], MAX_WINDOW) for k in range(len(bounds))]
    wins.append((edges[-1], int(np.max(in_end)), MAX_WINDOW))
    return wins


def water_fill(existing, expected, budget):
    """Skip spans per window for one endpoint (WaterFill, V3:863-917): raise the emptiest windows to a
    common level, capped by what each window still expects, then hand the remainder out one by one from
    the emptiest end.  `existing` / `expected` follow the windows sorted by start."""
    num = len(existing)
    alloc = np.zeros(num)
    if budget <= 0:
        return alloc
    existing = np.asarray(existing, np.float64)
    expected = np.asarray(expected, np.float64)
    order = np.argsort(existing)[::-1]          # the reference's call: its tie order is part of the result
    srt = existing[order]
    prefix = np.cumsum(srt)
    level, left = 0, 0
    for i in range(num):
        level = (budget + prefix[i]) // (i + 1)
        left = (budget + prefix[i]) % (i + 1)
        if level <= srt[i]:
            break
    want = np.maximum(level - srt, 0)
    room = expected - srt                      # (the reference pairs expected[i] with the i-th SORTED window)
    got = np.minimum(want, room)
    alloc[order] = got
    left += float(np.sum(want - got))
    while left > 0:
        changed = False
        for i in range(num - 1, -1, -1):
            if left > 0 and alloc[order[i]] < room[i]:
                alloc[order[i]] += 1
                left -= 1
                changed = True
        if not changed:
            break
    return alloc


def tally(in_start, in_end, sorted_out_start, state: SkipState):
    """TallySkipSpans, V3:853-989 (mutates state.time_windows like the reference).  Returns the windows
    sorted by start, the budgets and the per-ep, per-window skip counts."""
    state.time_windows.extend(new_time_windows(in_start, in_end))
    wins = sorted(state.time_windows, key=lambda w: w[0])
    ws = np.asarray([w[0] for w in wins], np.int64)
    we = np.asarray([w[1] for w in wins], np.int64)
    expected = [w[2] for w in wins]
    budgets = [len(in_start) - len(o) for o in sorted_out_start]
    counts = []
    for o, budget in zip(sorted_out_start, budgets):
        existing = np.searchsorted(o, we, side="right") - np.searchsorted(o, ws, side="right")   # ws < start <= we
        counts.append(np.maximum(water_fill(existing, expected, budget).astype(np.int64), 0).astype(np.int32))
    return wins, budgets, np.stack(counts)


def build_distributions(engine, in_start, in_end, sorted_out_start, sorted_out_end, labels, state: SkipState):
    """BuildDistributions, V3:108-172: the parent search on the device (tw_build_dist_samples), the
    sample lists and np.mean / np.std here.  labels = [incoming endpoint, out ep 0, ...].  Returns the
    dense [(E+1), (E+1), 2] table of services_times (NaN = no key)."""
    E = len(sorted_out_start)
    starts = np.concatenate([in_start] + list(sorted_out_start)).astype(np.int64)
    ends = np.concatenate([in_end] + list(sorted_out_end)).astype(np.int64)
    lab = np.concatenate([np.zeros(len(in_start), np.int8)] +
                         [np.full(len(o), 1 + e, np.int8) for e, o in enumerate(sorted_out_start)])
    order = np.argsort(starts, kind="stable")               # spans.sort(key=start_mus), V3:119
    starts, ends, lab = starts[order], ends[order], lab[order]
    large_delay = int(np.max(np.asarray(in_end, np.int64) - np.asarray(in_start, np.int64)))
    dev = engine.device
    d = _to_device(dict(start=starts, end=ends, label=lab), dev)
    key = torch.empty(len(starts), dtype=torch.int32, device=dev)
    val = torch.empty(len(starts), dtype=torch.int64, device=dev)
    _lib.check(engine.lib.tw_build_dist_samples(engine.h, len(starts), _p(d["start"]), _p(d["end"]), _p(d["label"]),
                                                E, C.c_int64(large_delay), _p(key), _p(val), engine.stream),
               "tw_build_dist_samples")
    key, val = key.cpu().numpy(), val.cpu().numpy()
    dv = state.distribution_values
    for k in np.unique(key[key >= 0]):
        a, b = divmod(int(k), E + 1)
        dv.setdefault((labels[a], labels[b]), []).extend(val[key == k].tolist())
    dv.setdefault((labels[0], labels[0]), []).extend((ends - starts)[lab == 0].tolist())      # V3:166-168
    tab = np.full((E + 1, E + 1, 2), np.nan)
    for a in range(E + 1):
        for b in range(E + 1):
            v = dv.get((labels[a], labels[b]))
            if v:
                tab[a, b] = (np.mean(v), np.std(v))
    return tab, large_delay


def sort_partitions(out_start, out_end):
    """TallySkipSpans sorts every partition by float(start), stable (V3:968-971).  Returns the
    permutations (sorted j -> caller's position) and the sorted arrays."""
    order = [np.argsort(np.asarray(o, np.int64).astype(np.float64), kind="stable") for o in out_start]
    s_start = [np.ascontiguousarray(np.asarray(o, np.int64)[od]) for o, od in zip(out_start, order)]
    s_end = [np.ascontiguousarray(np.asarray(o, np.int64)[od]) for o, od in zip(out_end, order)]
    return order, s_start, s_end


def marshal(in_start, in_end, s_start, s_end, order, preds, wins, counts, pair, budgets):
    """Host arrays of tw_batch + tw_skip_desc for ONE service (sorted lists + the caller's order)."""
    E = len(s_start)
    prob = Problem(in_start=in_start, in_end=in_end, out_start=s_start, out_end=s_end, preds=preds, name="skip")
    hb = build_batch([prob])
    n_win = len(wins)
    pred_order = np.full((E, _abi.TW_MAX_E), -1, np.int8)
    for e, pl in enumerate(preds):
        pred_order[e, :len(pl)] = pl
    entry_pos = np.concatenate(order).astype(np.int32)                       # sorted j -> caller's position
    sorted_of_entry = np.concatenate([np.argsort(od) for od in order]).astype(np.int32)
    host = dict(prob_win_off=np.array([0, n_win], np.int64), win_start=np.array([w[0] for w in wins], np.int64),
                prob_cnt_off=np.array([0, E * n_win], np.int64),
                skip_count=np.ascontiguousarray(np.asarray(counts).reshape(-1), np.int32),
                prob_pair_off=np.array([0, (E + 1) ** 2], np.int64),
                pair_gauss=np.ascontiguousarray(np.asarray(pair, np.float64).reshape(-1)),
                prob_normalized=np.array([1 if any(b > 0 for b in budgets) else 0], np.uint8),
                ep_pred_order=pred_order.reshape(-1), out_entry_pos=entry_pos, out_sorted_of_entry=sorted_of_entry)
    return hb, host


def to_caller_order(res, order, n, E, want_topk=True):
    """Result indices refer to the sorted lists: translate to positions in the caller's lists (codes < 0 stay)."""
    def conv(idx, ep_last):
        idx = idx.copy()
        for e in range(E):
            col = idx[..., e] if ep_last else idx[e]
            m = col >= 0
            col[m] = order[e][col[m]]
        return idx
    res["assign"] = conv(res["assign"].reshape(E, n), False)
    res["top2_idx"] = conv(res["top2_idx"].reshape(n, _abi.TW_K, E), True)
    if want_topk:
        res["topk_idx"] = conv(res["topk_idx"].reshape(n, _abi.TW_K, E), True)
    return res


def to_sorted_order(idx, order, ep_last):
    """Inverse of to_caller_order for one index array: positions in the caller's lists -> sorted-list
    indices.  Codes < 0 stay, and so does a position past the end of its list (scored as out of range)."""
    idx = np.array(idx, np.int32)
    for e, od in enumerate(order):
        col = idx[..., e] if ep_last else idx[e]
        m = (col >= 0) & (col < len(od))
        col[m] = np.argsort(od)[col[m]]
    return idx


def _descriptors(engine, hb, host):
    """Device copies of a marshalled service and the three structs tw_skip_solve and
    tw_skip_score_assignments take (the device arrays ride along: they must outlive the call)."""
    d = _to_device(host, engine.device)
    db = _to_device(hb.arrays, engine.device)
    return (batch_struct(hb, lambda name: db[name].data_ptr()), batch_struct(hb, lambda name: hb.arrays[name].ctypes.data),
            _abi.fill(_abi.TwSkipDesc, d), (d, db))


def _assess(engine, structs, n, assign, top2=None):
    """tw_skip_score_assignments of ONE service: device tensors score / code / margin (with `top2`, a
    TwSkipOut) per in-span, prob_sum [1], prob_count [1, TW_SKIP_ASSESS_NCODES]."""
    dev_struct, host_struct, sd, _ = structs
    dev = engine.device
    lk = dict(score=torch.empty(n, dtype=torch.float64, device=dev), code=torch.empty(n, dtype=torch.uint8, device=dev),
              prob_sum=torch.empty(1, dtype=torch.float64, device=dev),
              prob_count=torch.empty((1, _abi.TW_SKIP_ASSESS_NCODES), dtype=torch.int32, device=dev))
    if top2 is not None:
        lk["margin"] = torch.empty(n, dtype=torch.float64, device=dev)
    _lib.check(engine.lib.tw_skip_score_assignments(
        engine.h, C.byref(dev_struct), C.byref(host_struct), C.byref(sd), _p(assign),
        C.byref(top2) if top2 is not None else None, _p(lk["score"]), _p(lk["code"]), _p(lk.get("margin")),
        _p(lk["prob_sum"]), _p(lk["prob_count"]), engine.stream), "tw_skip_score_assignments")
    return lk


def _likelihood(lk):
    res = dict(chosen_score=lk["score"].cpu().numpy(), chosen_code=lk["code"].cpu().numpy(),
               service_score=float(lk["prob_sum"][0]), service_codes=lk["prob_count"][0].cpu().numpy())
    if "margin" in lk:
        res["margin"] = lk["margin"].cpu().numpy()
    return res


def solve(engine, in_start, in_end, out_start, out_end, preds, labels=None, state: SkipState = None,
          want_topk=True, want_likelihood=False):
    """One FindAssignments call in the skip regime for ONE service.  out_start/out_end: per ep
    (topological order) in the CALLER's list order.  Returns numpy arrays; out spans are named by their
    position in the caller's lists, skip spans by -2 - g (see include/traceweaver_b200.h), ("Skip", "Skip")
    assignments by -2, ("NA", "NA") by -1.

    want_likelihood: also how sure the engine is of each choice.  Its final assignment is scored under the
    model it solved with (tw_skip_score_assignments) and compared with the in-span's top2 list:
        chosen_score   float64 [n]  the tuple's score, NaN unless scored.  Where some budget is positive
                                    (the normal case here) a MEAN OF DENSITIES, not a log-likelihood:
                                    not comparable with the two-pass regime's scores
        chosen_code    uint8   [n]  TW_ASSESS_* / TW_SKIP_ASSESS_UNDEFINED (1 = unassigned)
        margin         float64 [n]  chosen = rank 0: s0 - s1 (+inf: single candidate), else score - s0
        service_score  float        sum of the scored in-spans' scores
        service_codes  int32   [6]  in-spans per code"""
    state = state if state is not None else SkipState()
    E = len(out_start)
    labels = labels or list(range(E + 1))
    in_start = np.ascontiguousarray(in_start, np.int64)
    in_end = np.ascontiguousarray(in_end, np.int64)
    order, s_start, s_end = sort_partitions(out_start, out_end)
    wins, budgets, counts = tally(in_start, in_end, s_start, state)
    pair, large_delay = build_distributions(engine, in_start, in_end, s_start, s_end, labels, state)
    hb, host = marshal(in_start, in_end, s_start, s_end, order, preds, wins, counts, pair, budgets)
    dev = engine.device
    n, nt = len(in_start), len(in_start) * E
    structs = _descriptors(engine, hb, host)
    dev_struct, host_struct, sd, _ = structs
    out = dict(assign=torch.empty(nt, dtype=torch.int32, device=dev), mis_rank=torch.empty(n, dtype=torch.int8, device=dev),
               n_cand=torch.empty(n, dtype=torch.int32, device=dev), counters=torch.zeros((1, 4), dtype=torch.int32, device=dev),
               top2_score=torch.empty((n, _abi.TW_K), dtype=torch.float64, device=dev),
               top2_idx=torch.empty(_abi.TW_K * nt, dtype=torch.int32, device=dev),
               top2_cnt=torch.empty(n, dtype=torch.uint8, device=dev), cut=torch.empty(n, dtype=torch.uint8, device=dev))
    if want_topk:
        out.update(topk_score=torch.empty((n, _abi.TW_K), dtype=torch.float64, device=dev),
                   topk_idx=torch.empty(_abi.TW_K * nt, dtype=torch.int32, device=dev),
                   topk_cnt=torch.empty(n, dtype=torch.uint8, device=dev))
    so = _abi.fill(_abi.TwSkipOut, out)
    _lib.check(engine.lib.tw_skip_solve(engine.h, C.byref(dev_struct), C.byref(host_struct), C.byref(sd), C.byref(so),
                                        engine.stream), "tw_skip_solve")
    lk = _assess(engine, structs, n, out["assign"], top2=so) if want_likelihood else None
    engine.status()
    res = to_caller_order({k: v.cpu().numpy() for k, v in out.items()}, order, n, E, want_topk)
    res.update(time_windows=wins, skip_budget=budgets, skip_count=counts, pair_params=pair, large_delay=large_delay,
               sorted_order=order)
    if want_likelihood:
        res.update(_likelihood(lk))
    return res


def score(engine, in_start, in_end, out_start, out_end, preds, assign, state_snapshot):
    """The score of ANY assignment of a cache-mode service (the engine's, the ground truth, another
    predictor's) under the model an earlier `solve` of that service used.  in_start ... preds as given
    to `solve`; assign [E, n] in the caller's list positions, -1 = ("NA", "NA"), <= -2 = ("Skip", "Skip")
    (which skip span does not matter); state_snapshot: the dict that `solve` returned (its pair table,
    budgets, which decide `normalized`, windows and skip counts; with its top2 lists the margin too).
    Returns host arrays score / code [n] (code TW_ASSESS_* / TW_SKIP_ASSESS_UNDEFINED, score NaN unless
    code 0), margin [n] when the snapshot has top2 lists, service_score, service_codes [6]."""
    E, n = len(out_start), len(in_start)
    assign = np.asarray(assign, np.int32)
    if assign.shape != (E, n):
        raise ValueError(f"score: assign must have shape ({E}, {n})")
    in_start = np.ascontiguousarray(in_start, np.int64)
    in_end = np.ascontiguousarray(in_end, np.int64)
    snap = state_snapshot
    order, s_start, s_end = sort_partitions(out_start, out_end)
    hb, host = marshal(in_start, in_end, s_start, s_end, order, preds, snap["time_windows"], snap["skip_count"],
                       snap["pair_params"], snap["skip_budget"])
    structs = _descriptors(engine, hb, host)
    top2 = None
    if "top2_idx" in snap:
        t2 = _to_device(dict(top2_score=np.ascontiguousarray(snap["top2_score"], np.float64),
                             top2_idx=to_sorted_order(snap["top2_idx"], order, True).reshape(-1),
                             top2_cnt=np.ascontiguousarray(snap["top2_cnt"], np.uint8)), engine.device)
        top2 = _abi.fill(_abi.TwSkipOut, t2)
    a = _to_device(dict(assign=to_sorted_order(assign, order, False).reshape(-1)), engine.device)["assign"]
    lk = _assess(engine, structs, n, a, top2)
    engine.status()
    res = _likelihood(lk)
    return dict(score=res.pop("chosen_score"), code=res.pop("chosen_code"), **res)
