"""Host-side problem/batch descriptors: the SoA layout the engine consumes.

A *problem* is what the reference hands to `TraceWeaverV3.FindAssignments`
(executor.py:1172-1175): the spans arriving at one service (one incoming endpoint) and the spans
it sends to each outgoing endpoint, plus the invocation DAG over the outgoing endpoints.  Here it
is index-only: microsecond start/end arrays sorted by (start, end) (executor.py:1111-1112),
endpoints in topological order (traceweaver_v1.py:37-39), DAG as predecessor lists in
`in_edges` order (the order the reference sums likelihood terms in, traceweaver_v1.py:322).

`build_batch` concatenates problems into the arrays of `tw_batch` (include/traceweaver_b200.h).
Times are int64 microseconds, or float64 microseconds for time-compressed spans (executor.py
--compress_factor > 1 divides start times by the factor): a batch in which any span array has a
floating dtype is a float64 batch, and the engine binds it through tw_engine_bind_f64.
Pure numpy; no device code here.
"""
from dataclasses import dataclass, field
from typing import List, Sequence

import numpy as np

from . import _abi

SPAN_ARRAYS = ("in_start", "in_end", "out_start", "out_end")


def _time_dtype(arrays):
    """float64 if any of the span arrays has a floating dtype, else int64."""
    return np.float64 if any(np.asarray(a).dtype.kind == "f" for a in arrays) else np.int64


@dataclass
class Problem:
    in_start: np.ndarray                 # int64 or float64 [n_in]
    in_end: np.ndarray                   # int64 or float64 [n_in]
    out_start: List[np.ndarray]          # per ep (topological order): int64 or float64 [n_out_e]
    out_end: List[np.ndarray]
    preds: List[List[int]]               # per ep: predecessor positions, in_edges order
    name: str = ""

    @property
    def E(self):
        return len(self.out_start)

    @property
    def n_in(self):
        return int(self.in_start.shape[0])

    def is_primary(self, b, e):
        """Edge b->e is NON-primary iff a 2-hop path b->x->e exists
        (AlsoNonPrimaryAncestor, traceweaver_v1.py:294-303: all_simple_paths(cutoff=2))."""
        for x in range(self.E):
            if x != b and x != e and b in self.preds[x] and x in self.preds[e]:
                return False
        return True

    def terms(self):
        """[(ep, src)] in the reference's summation order (traceweaver_v1.py:316-357):
        per ep: primary in-edges in in_edges order | ROOT if no in-edges; then LAST."""
        out = []
        for e in range(self.E):
            for b in self.preds[e]:
                if self.is_primary(b, e):
                    out.append((e, b))
            if len(self.preds[e]) == 0:
                out.append((e, _abi.TW_TERM_ROOT))
            out.append((e, _abi.TW_TERM_LAST))
        return out

    def validate(self):
        E = self.E
        if not (1 <= E <= _abi.TW_MAX_E):
            raise ValueError(f"{self.name}: E={E} outside [1, {_abi.TW_MAX_E}]")
        if self.n_in < 2:
            # the reference builds no window for a single in-span and then fails on max([])
            # (traceweaver_v3.py:1056-1076, :1119)
            raise ValueError(f"{self.name}: need at least 2 incoming spans")
        for e in range(E):
            for b in self.preds[e]:
                if not (0 <= b < e):
                    raise ValueError(f"{self.name}: preds must reference earlier topological positions")
        if len(self.out_end) != E or len(self.preds) != E:
            raise ValueError(f"{self.name}: out_start / out_end / preds must have one entry per ep")
        if self.in_end.shape != self.in_start.shape:
            raise ValueError(f"{self.name}: in_start and in_end differ in length")
        if np.any(self.in_end < self.in_start):
            raise ValueError(f"{self.name}: an in-span ends before it starts")
        key = self.in_start if self.in_start.dtype.kind == "f" else self.in_start.astype(np.int64)
        if np.any(np.diff(key) < 0):
            raise ValueError(f"{self.name}: in-spans not sorted by start")
        for e in range(E):
            if self.out_end[e].shape != self.out_start[e].shape:
                raise ValueError(f"{self.name}: out_start and out_end of ep {e} differ in length")
            if np.any(self.out_end[e] < self.out_start[e]):
                raise ValueError(f"{self.name}: an out-span of ep {e} ends before it starts")
            if np.any(np.diff(self.out_start[e]) < 0):
                raise ValueError(f"{self.name}: out-spans of ep {e} not sorted by start")

    def in_accelerated_regime(self):
        """True iff every ep has as many outgoing spans as there are incoming ones (no skip budget,
        traceweaver_v3.py:1138-1158): the regime the engine solves."""
        return all(len(o) == self.n_in for o in self.out_start)


@dataclass
class HostBatch:
    problems: Sequence[Problem]
    arrays: dict = field(default_factory=dict)

    def __getattr__(self, k):
        try:
            return self.__dict__["arrays"][k]
        except KeyError:
            raise AttributeError(k)

    @property
    def n_problems(self):
        return len(self.problems)

    @property
    def float_times(self):
        """True for a batch of float64 microsecond times (bound through tw_engine_bind_f64)."""
        return self.arrays["in_start"].dtype == np.float64

    def no_skip(self):
        """True iff every ep of every problem has n_out == n_in (the regime with two passes,
        traceweaver_v3.py:1138-1158)."""
        a = self.arrays
        n_in = np.diff(a["prob_in_off"])
        n_out = np.diff(a["ep_out_off"])
        ep_prob = np.repeat(np.arange(self.n_problems), np.diff(a["prob_ep_off"]))
        return bool(np.all(n_out == n_in[ep_prob]))

    def slice(self, lo: int, hi: int) -> "HostBatch":
        """Sub-batch of problems [lo, hi): offset tables rebased, span arrays are views (no copy).
        Services are independent problems, so solving the slices separately gives the same result."""
        a = self.arrays
        e0, e1 = int(a["prob_ep_off"][lo]), int(a["prob_ep_off"][hi])
        t0, t1 = int(a["ep_term_off"][e0]), int(a["ep_term_off"][e1])
        i0, i1 = int(a["prob_in_off"][lo]), int(a["prob_in_off"][hi])
        o0, o1 = int(a["ep_out_off"][e0]), int(a["ep_out_off"][e1])

        def reb(name, x0, x1):
            v = a[name][x0:x1 + 1]
            return np.ascontiguousarray(v - v[0])

        arrays = dict(
            prob_in_off=reb("prob_in_off", lo, hi), prob_ep_off=reb("prob_ep_off", lo, hi),
            prob_tuple_off=reb("prob_tuple_off", lo, hi), ep_out_off=reb("ep_out_off", e0, e1),
            ep_term_off=reb("ep_term_off", e0, e1), ep_pred_mask=a["ep_pred_mask"][e0:e1],
            term_src=a["term_src"][t0:t1], in_start=a["in_start"][i0:i1], in_end=a["in_end"][i0:i1],
            out_start=a["out_start"][o0:o1], out_end=a["out_end"][o0:o1],
            prob_gauss_off=reb("prob_gauss_off", lo, hi), term_sample_off=reb("term_sample_off", t0, t1))
        probs = self.problems[lo:hi] if isinstance(self.problems, list) else _ProblemCount(hi - lo)
        return HostBatch(problems=probs, arrays=arrays)


def _cumulative(counts, dtype):
    return np.concatenate([[0], np.cumsum(counts)]).astype(dtype)


def offset_tables(n_in, E, n_out, n_term=None):
    """The offset tables of tw_batch from the counts: n_in and E per problem, n_out per ep (problem by
    problem, topological order).  With n_term (terms per ep) also the term tables: ep_term_off,
    prob_gauss_off (one record per term and 100-span batch) and term_sample_off (a term holds up to
    n_in samples of its problem, tw_delays)."""
    n_in = np.asarray(n_in, np.int64)
    E = np.asarray(E, np.int64)
    t = dict(prob_in_off=_cumulative(n_in, np.int64), prob_ep_off=_cumulative(E, np.int32),
             prob_tuple_off=_cumulative(n_in * E, np.int64), ep_out_off=_cumulative(n_out, np.int64))
    if n_term is not None:
        t["ep_term_off"] = _cumulative(n_term, np.int32)
        prob_terms = np.diff(t["ep_term_off"].astype(np.int64)[t["prob_ep_off"]])
        n_batches = (n_in + _abi.TW_PARAM_BATCH - 1) // _abi.TW_PARAM_BATCH
        t["prob_gauss_off"] = _cumulative(n_batches * prob_terms, np.int64)
        t["term_sample_off"] = _cumulative(np.repeat(n_in, prob_terms), np.int64)
    return t


def build_batch(problems: Sequence[Problem], validate=True) -> HostBatch:
    if len(problems) == 0:
        raise ValueError("empty batch")
    if validate:
        for p in problems:
            p.validate()
    n_out, n_term, ep_pred_mask, term_src = [], [], [], []
    for p in problems:
        terms = p.terms()
        for e in range(p.E):
            n_out.append(int(p.out_start[e].shape[0]))
            mask = 0
            for b in p.preds[e]:
                mask |= 1 << b
            ep_pred_mask.append(mask)
            mine = [src for (ee, src) in terms if ee == e]
            term_src.extend(mine)
            n_term.append(len(mine))
    tdt = _time_dtype([a for p in problems for a in [p.in_start, p.in_end] + list(p.out_start) + list(p.out_end)])
    arrays = offset_tables([p.n_in for p in problems], [p.E for p in problems], n_out, n_term)
    arrays.update(
        ep_pred_mask=np.asarray(ep_pred_mask, np.uint32), term_src=np.asarray(term_src, np.int8),
        in_start=np.ascontiguousarray(np.concatenate([p.in_start for p in problems]), tdt),
        in_end=np.ascontiguousarray(np.concatenate([p.in_end for p in problems]), tdt),
        out_start=np.ascontiguousarray(np.concatenate([s for p in problems for s in p.out_start]), tdt),
        out_end=np.ascontiguousarray(np.concatenate([s for p in problems for s in p.out_end]), tdt),
    )
    return HostBatch(problems=list(problems), arrays=arrays)


def batch_struct(hb: HostBatch, ptr):
    """Fill a TwBatch with pointers produced by `ptr(name)` (host or device).  A batch without term
    tables (truth.TraceLists) gets NULL ep_term_off / ep_pred_mask / term_src and n_term_total = 0."""
    a = hb.arrays
    s = _abi.TwBatch(n_problems=hb.n_problems, n_ep_total=int(a["prob_ep_off"][-1]),
                     n_term_total=int(a["ep_term_off"][-1]) if "ep_term_off" in a else 0,
                     n_in_total=int(a["prob_in_off"][-1]), n_out_total=int(a["ep_out_off"][-1]))
    for name, typ in _abi.TwBatch._fields_:
        if typ is _abi.P and name in a:
            setattr(s, name, ptr(name))
    return s


@dataclass
class ServiceBlock:
    """S services with identical shape (n_in, E, DAG): the vectorised form used by the synthetic
    generators.  Arrays are [S, n]; out lists are per ep in topological order."""
    in_start: np.ndarray
    in_end: np.ndarray
    out_start: List[np.ndarray]
    out_end: List[np.ndarray]
    preds: List[List[int]]
    truth: np.ndarray = None            # [E, S, n] index of the true child in each ep list
    name: str = ""

    def problem(self, s) -> Problem:
        return Problem(in_start=self.in_start[s], in_end=self.in_end[s],
                       out_start=[o[s] for o in self.out_start], out_end=[o[s] for o in self.out_end],
                       preds=self.preds, name=f"{self.name}[{s}]")


def build_batch_from_blocks(blocks: Sequence[ServiceBlock]) -> HostBatch:
    """Same arrays as build_batch([...problems of every block...]) without per-problem Python work."""
    n_in, n_ep, n_out, n_term, ep_pred, term_src = [], [], [], [], [], []
    ins, ine, outs, oute = [], [], [], []
    for blk in blocks:
        S, n = blk.in_start.shape
        E = len(blk.out_start)
        tmpl = Problem(in_start=blk.in_start[0], in_end=blk.in_end[0], out_start=[o[0] for o in blk.out_start],
                       out_end=[o[0] for o in blk.out_end], preds=blk.preds, name=blk.name)
        tmpl.validate()
        terms = tmpl.terms()
        per_ep_terms = [[src for (ee, src) in terms if ee == e] for e in range(E)]
        masks = [sum(1 << b for b in blk.preds[e]) for e in range(E)]
        n_in.append(np.full(S, n))
        n_ep.append(np.full(S, E))
        n_out.append(np.full(S * E, n))
        n_term.append(np.tile([len(t) for t in per_ep_terms], S))
        ep_pred.extend(masks * S)
        term_src.extend([src for t in per_ep_terms for src in t] * S)
        ins.append(blk.in_start.reshape(-1))
        ine.append(blk.in_end.reshape(-1))
        # per problem: ep 0 list, ep 1 list, ...  -> stack [S, E, n]
        outs.append(np.stack(blk.out_start, axis=1).reshape(-1))
        oute.append(np.stack(blk.out_end, axis=1).reshape(-1))
    tdt = _time_dtype(ins + ine + outs + oute)
    arrays = offset_tables(np.concatenate(n_in), np.concatenate(n_ep), np.concatenate(n_out), np.concatenate(n_term))
    arrays.update(
        ep_pred_mask=np.asarray(ep_pred, np.uint32), term_src=np.asarray(term_src, np.int8),
        in_start=np.ascontiguousarray(np.concatenate(ins), tdt),
        in_end=np.ascontiguousarray(np.concatenate(ine), tdt),
        out_start=np.ascontiguousarray(np.concatenate(outs), tdt),
        out_end=np.ascontiguousarray(np.concatenate(oute), tdt))
    return HostBatch(problems=_ProblemCount(len(arrays["prob_in_off"]) - 1), arrays=arrays)


class _ProblemCount:
    """len()-only stand-in for the problem list of a block-built batch."""

    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n
