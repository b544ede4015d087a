"""Synthetic cache-mode services for the skip regime's tests (test infrastructure only).

A service starts as a `traceweaver_b200.synth.make_block` service (or, for the eight-callee DAG that no
shipped shape has, the same laws on a DAG: a callee starts after the last of its predecessors ends).
Cache hits are then modelled the way the reference's cache transform (helpers/transforms.py,
create_cache_hits) makes them: the cached call's span is dropped, every later span of that trace moves
earlier by the cached call's duration, the incoming span ends that much earlier, and the lists are NOT
re-sorted afterwards, so they arrive partly out of order.  `extra` adds spans that belong to no trace
(more outgoing than incoming spans: a negative skip budget).

`run_oracle` runs `oracle/tw_oracle_skip.solve_skip` with its branches counted (sys.monitoring on the
oracle's own code objects, nothing in the oracle changes), so the tests can say which branches the
generated inputs reach.

`dag_problem` builds two-pass services (no cache hits) on the DAGs of DAG_SHAPES with the same laws,
for the tests of services with five to eight callees (tests/test_dag_shapes.py).
"""
import inspect
import sys
from dataclasses import dataclass, field

import numpy as np

from oracle import tw_oracle_skip as osk
from traceweaver_b200 import _abi, synth

SHAPES = sorted(synth.SHAPES)
# two chains (0-1-2-3 and 4-5-6) joining at 7; the edge 2 -> 7 is transitive through 3 (non-primary)
DAG8 = dict(preds=[[], [0], [1], [2], [], [4], [5], [3, 6, 2]],
            eps=[(300, 0.6, 1500, 0.5)] * 8, tail=(200, 0.6), ia100=33_300.0)


@dataclass
class SkipService:
    name: str
    in_start: np.ndarray
    in_end: np.ndarray
    out_start: list                  # per callee, the caller's order (partly unsorted after cache hits)
    out_end: list
    preds: list
    truth: np.ndarray                # [E, n]: position in the caller's list, -2 where the call was cached
    wins_before: list = field(default_factory=list)
    values_before: dict = field(default_factory=dict)

    @property
    def E(self):
        return len(self.out_start)

    @property
    def n(self):
        return len(self.in_start)


def dag_trace_times(spec, n, load, seed, quantum):
    """make_block's laws on a DAG: [n] in-span times, per-callee [n] span times of trace i."""
    rng = np.random.default_rng(seed)
    ia = np.maximum(np.rint(rng.exponential(spec["ia100"] * 100.0 / load, size=n)), 1).astype(np.int64)
    in_s = synth.T0 + np.cumsum(ia)
    starts, ends = [], []
    for e, (gm, gs, dm, ds) in enumerate(spec["eps"]):
        base = in_s.copy()
        for b in spec["preds"][e]:
            base = np.maximum(base, ends[b])
        s = base + synth._lognormal(rng, gm, gs, n)
        starts.append(s)
        ends.append(s + synth._lognormal(rng, dm, ds, n))
    in_e = np.max(ends, axis=0) + synth._lognormal(rng, spec["tail"][0], spec["tail"][1], n)
    q = quantum
    return in_s // q * q, in_e // q * q, [s // q * q for s in starts], [x // q * q for x in ends]


def _traces(shape, n, load, seed, quantum):
    """(in_s, in_e, starts [E][n], ends [E][n], preds) with trace i's call of callee e at [e][i]."""
    if shape == "dag8":
        in_s, in_e, st, en = dag_trace_times(DAG8, n, load, seed, quantum)
        o = np.lexsort((in_e, in_s))
        return in_s[o], in_e[o], [s[o] for s in st], [x[o] for x in en], DAG8["preds"]
    blk = synth.make_block(shape, 1, n_in=n, load=load, seed=seed, quantum_us=quantum)
    tr = blk.truth[:, 0, :]
    st = [blk.out_start[e][0][tr[e]] for e in range(len(blk.out_start))]
    en = [blk.out_end[e][0][tr[e]] for e in range(len(blk.out_start))]
    return blk.in_start[0].copy(), blk.in_end[0].copy(), st, en, blk.preds


# Two-pass services on DAGs no synth.SHAPES entry has (predecessor lists in in_edges order, which is the
# order the score sums a callee's edge terms in): name -> (preds, number of score terms)
_EPS, _TAIL = DAG8["eps"][0], DAG8["tail"]
DAG_SHAPES = {
    "dag8": (DAG8["preds"], 17),
    # K4,4: four parallel roots, four sinks after all of them (in scrambled in_edges order): the most
    # terms a service of eight callees can have (4 roots + 16 edges + 8 lasts)
    "k44": ([[], [], [], [], [3, 1, 0, 2], [0, 1, 2, 3], [2, 3, 1, 0], [1, 0, 3, 2]], 28),
    "k33": ([[], [], [], [2, 0, 1], [1, 2, 0], [0, 1, 2]], 18),
    "mix7": ([[], [], [0], [0, 1], [3], [2, 4], [5, 1]], 17),
    "dag5": ([[], [0], [0], [2, 1], [1]], 11),
    # every callee after the one and the two before it: each transitive edge e-2 -> e is non-primary
    "chain8": ([[]] + [[e - 1] + ([e - 2] if e >= 2 else []) for e in range(1, 8)], 16),
    "diamond": ([[], [0], [0], [2, 1, 0]], 9),
}


def dag_problem(shape, n=260, ia_us=12_000.0, seed=0, quantum=1):
    """One two-pass service of DAG_SHAPES[shape] (batch.Problem) and its truth [E, n] (position of trace
    i's call in callee e's list): `n` in-spans with a mean inter-arrival of `ia_us`, timestamps rounded
    down to `quantum` us, in-spans and callee lists in (start, end) order like synth.make_block's."""
    from traceweaver_b200.batch import Problem
    preds = DAG_SHAPES[shape][0]
    E = len(preds)
    spec = dict(preds=preds, eps=[_EPS] * E, tail=_TAIL, ia100=ia_us)
    in_s, in_e, st, en = dag_trace_times(spec, n, 100.0, seed, quantum)
    o = np.lexsort((in_e, in_s))
    in_s, in_e, st, en = in_s[o], in_e[o], [s[o] for s in st], [x[o] for x in en]
    out_s, out_e = [], []
    truth = np.empty((E, n), np.int32)
    for e in range(E):
        od = np.lexsort((en[e], st[e]))
        truth[e, od] = np.arange(n)
        out_s.append(np.ascontiguousarray(st[e][od]))
        out_e.append(np.ascontiguousarray(en[e][od]))
    prob = Problem(in_start=np.ascontiguousarray(in_s), in_end=np.ascontiguousarray(in_e), out_start=out_s,
                   out_end=out_e, preds=[list(p) for p in preds], name=f"{shape}-n{n}-ia{ia_us:g}-s{seed}-q{quantum}")
    return prob, truth


def make_service(shape, n=120, load=60.0, seed=0, cached=(), rate=0.0, quantum=1, extra=(), shift=0):
    """One cache-mode service.  cached: callees whose calls hit the cache, each with probability `rate`
    per trace; quantum: clock grid in us (1000: millisecond clocks); extra: ((callee, count), ...) spans
    outside every trace; shift: added to every timestamp (to line services up on a common start)."""
    in_s, in_e, st, en, preds = _traces(shape, n, load, seed, quantum)
    E = len(st)
    rng = np.random.default_rng(seed * 7919 + 17)
    st = [s.copy() for s in st]
    en = [x.copy() for x in en]
    # the executor's (start, end) order first; extras are spans of other callers, sorted in with the rest
    recs = []
    for e in range(E):
        items = [(int(st[e][i]), int(en[e][i]), i) for i in range(n)]
        for ee, cnt in extra:
            if ee != e:
                continue
            for _ in range(cnt):
                i = int(rng.integers(n))
                lo, hi = int(in_s[i]), int(in_e[i])
                s = lo + int(rng.integers(0, max(1, (hi - lo) // 2)))
                x = min(hi, s + int(rng.integers(0, max(1, (hi - s)))))
                items.append((s // quantum * quantum, x // quantum * quantum, -1))
        items.sort(key=lambda r: (r[0], r[1]))
        recs.append(items)
    pos = [{r[2]: j for j, r in enumerate(items) if r[2] >= 0} for items in recs]
    s_cur = [[r[0] for r in items] for items in recs]
    e_cur = [[r[1] for r in items] for items in recs]
    dropped = np.zeros((E, n), bool)
    in_e = in_e.copy()
    for i in range(n):
        for e in sorted(cached, key=lambda c: s_cur[c][pos[c][i]]):
            if rng.random() >= rate:
                continue
            j = pos[e][i]
            cs, ce = s_cur[e][j], e_cur[e][j]
            delta = ce - cs
            dropped[e, i] = True
            for f in range(E):
                if dropped[f, i]:
                    continue
                k = pos[f][i]
                if s_cur[f][k] >= ce:
                    s_cur[f][k] -= delta
                    e_cur[f][k] -= delta
            live_end = max([e_cur[f][pos[f][i]] for f in range(E) if not dropped[f, i]], default=int(in_s[i]))
            in_e[i] = max(int(in_e[i]) - delta, live_end)
    out_start, out_end = [], []
    truth = np.full((E, n), -2, np.int32)
    for e in range(E):
        keep = [j for j, r in enumerate(recs[e]) if not (r[2] >= 0 and dropped[e, r[2]])]
        new = {j: k for k, j in enumerate(keep)}
        out_start.append(np.array([s_cur[e][j] for j in keep], np.int64) + shift)
        out_end.append(np.array([e_cur[e][j] for j in keep], np.int64) + shift)
        for i in range(n):
            if not dropped[e, i]:
                truth[e, i] = new[pos[e][i]]
    name = (f"{shape}-n{n}-L{load:g}-s{seed}-q{quantum}-c{''.join(map(str, cached)) or 'none'}@{rate:g}"
            f"-x{'.'.join(f'{a}x{b}' for a, b in extra) or 'none'}")
    return SkipService(name=name, in_start=in_s + shift, in_end=in_e + shift, out_start=out_start, out_end=out_end,
                       preds=[list(p) for p in preds], truth=truth)


# -------------------------------------------------------------------------------------------------
# the oracle, with its branches counted
# -------------------------------------------------------------------------------------------------
BRANCHES = {   # name -> (a piece of an oracle line, offset of the line that IS the branch)
    "skip_pred_root": ("# FindValidAncestor -> None", 1),
    "skip_pred_ancestor": ("(sic) the ancestor's START", 0),
    "err_ancestor_chain": ('"ancestor chain of skip spans"', 0),
    "tie_real_real": ("return sa < sb", 0),
    "err_tie_skip_real": ('"score tie between a skip span and a real span"', 0),
    "err_all_skip": ('"all-skip tuple"', 0),
    "err_missing_key": ('"no distribution for the pair', 0),
    "err_no_window": ('"no time window starts at or before', 0),
    "non_primary_edge": ("if not primary(b, e):", 1),
}


class _BranchCounter:
    def __init__(self):
        src = inspect.getsource(osk).splitlines()
        self.lines = {}
        for name, (marker, offset) in BRANCHES.items():
            hits = [k + 1 for k, line in enumerate(src) if marker in line]
            assert len(hits) == 1, (name, hits)
            self.lines[hits[0] + offset] = name
        self.codes = []

        def walk(co):
            self.codes.append(co)
            for c in co.co_consts:
                if inspect.iscode(c):
                    walk(c)
        walk(osk.solve_skip.__code__)
        walk(osk._Entry.__lt__.__code__)
        self.counts = None

    def _on_line(self, code, line):
        name = self.lines.get(line)
        if name is None:
            return sys.monitoring.DISABLE
        self.counts[name] = self.counts.get(name, 0) + 1
        return None

    def run(self, fn):
        mon = sys.monitoring
        tool = next(t for t in range(6) if mon.get_tool(t) is None)
        mon.use_tool_id(tool, "skip_synth branch counter")
        self.counts = {}
        try:
            mon.register_callback(tool, mon.events.LINE, self._on_line)
            for co in self.codes:
                mon.set_local_events(tool, co, mon.events.LINE)
            try:
                return fn(), dict(self.counts)
            except osk.ReferenceUndefined as ex:
                return ex, dict(self.counts)
        finally:
            for co in self.codes:
                mon.set_local_events(tool, co, 0)
            mon.register_callback(tool, mon.events.LINE, None)
            mon.free_tool_id(tool)
            mon.restart_events()


_COUNTER = None


def model(svc):
    """The skip regime's model of a service from the oracle's own pieces: windows, budgets, skip counts,
    the services_times table (with the samples of earlier services) and the new samples."""
    order = [sorted(range(len(o)), key=lambda j, o=o: float(o[j])) for o in svc.out_start]
    s_start = [[int(o[j]) for j in od] for o, od in zip(svc.out_start, order)]
    s_end = [[int(o[j]) for j in od] for o, od in zip(svc.out_end, order)]
    ins, ine = [int(x) for x in svc.in_start], [int(x) for x in svc.in_end]
    wins, budgets, counts = osk.tally_skip_spans(ins, ine, s_start, list(svc.wins_before))
    samples, _ = osk.build_distribution_samples(ins, ine, s_start, s_end)
    tab = osk.pair_params(samples, svc.E, svc.values_before)
    return dict(wins=wins, budgets=budgets, counts=counts, tab=tab, samples=samples,
                normalized=any(b > 0 for b in budgets))


def run_oracle(svc):
    """(solve_skip's result dict or the ReferenceUndefined it raised, branch counts, model)."""
    global _COUNTER
    if _COUNTER is None:
        _COUNTER = _BranchCounter()
    res, counts = _COUNTER.run(lambda: osk.solve_skip(svc.in_start, svc.in_end, svc.out_start, svc.out_end,
                                                      svc.preds, time_windows_before=list(svc.wins_before),
                                                      values_before=svc.values_before))
    return res, counts, model(svc)


def input_features(svc, md):
    """Properties of the input the table of reached branches reports beside the oracle's counts."""
    f = {}
    f[f"E={svc.E}"] = 1
    f["normalized=0"] = int(not md["normalized"])
    f["mixed budget signs"] = int(any(b > 0 for b in md["budgets"]) and any(b < 0 for b in md["budgets"]))
    f["unsorted caller list"] = int(any(np.any(np.diff(o) < 0) for o in svc.out_start))
    f["equal starts in a list"] = int(any(np.any(np.diff(np.sort(o)) == 0) for o in svc.out_start))
    ws = [w[0] for w in md["wins"]]
    shared = {s for s in ws if ws.count(s) > 1}
    f["in-span in a window with a shared start"] = 0
    for s in svc.in_start:
        c = [x for x in ws if x <= s]
        if c and max(c) in shared:
            f["in-span in a window with a shared start"] += 1
    return f


def cand_limit_service(n_cand, E=2, seed=0):
    """One long in-span holding `n_cand` spans of callee 0 (and one of every other callee), between
    short ordinary in-spans: the per-in-span candidate limit of the skip search."""
    rng = np.random.default_rng(seed)
    n = 12
    in_s = synth.T0 + np.arange(n, dtype=np.int64) * 100_000
    in_e = in_s + 20_000
    in_e[5] = in_s[5] + 300_000
    out_s, out_e = [], []
    truth = np.full((E, n), -2, np.int32)
    for e in range(E):
        s = in_s + 1_000 + 500 * e
        x = s + 2_000
        if e == 0:
            extra_s = in_s[5] + 10_000 + np.sort(rng.integers(0, 250_000, n_cand - 3))   # + own and 2 later traces
            extra_e = extra_s + rng.integers(100, 30_000, n_cand - 3)
            extra_e = np.minimum(extra_e, in_e[5] - 1)
            s = np.concatenate([s, extra_s])
            x = np.concatenate([x, extra_e])
        od = np.lexsort((x, s))
        inv = np.empty_like(od)
        inv[od] = np.arange(len(od))
        truth[e] = inv[:n]
        out_s.append(s[od])
        out_e.append(x[od])
    return SkipService(name=f"candlimit{n_cand}-E{E}", in_start=in_s, in_end=in_e, out_start=out_s, out_end=out_e,
                       preds=[[]] * E, truth=truth)


def with_history(svc, prior):
    """`svc` as the second service a predictor instance sees, `prior` (same callee count) first: prior's
    time windows and distribution samples come before, and prior is moved in time so that both services
    open a window at the same start (FetchSkipFromWindow then takes the first of the equal starts)."""
    d = int(svc.in_start[0]) - int(prior.in_start[0])
    ps, pe = [int(x) + d for x in prior.in_start], [int(x) + d for x in prior.in_end]
    order = [sorted(range(len(o)), key=lambda j, o=o: float(o[j])) for o in prior.out_start]
    os_ = [[int(o[j]) + d for j in od] for o, od in zip(prior.out_start, order)]
    oe_ = [[int(o[j]) + d for j in od] for o, od in zip(prior.out_end, order)]
    values = {}
    for k, v in osk.build_distribution_samples(ps, pe, os_, oe_)[0]:
        values.setdefault(k, []).append(v)
    return SkipService(name=f"{svc.name}-after-{prior.name}", in_start=svc.in_start, in_end=svc.in_end,
                       out_start=svc.out_start, out_end=svc.out_end, preds=svc.preds, truth=svc.truth,
                       wins_before=list(svc.wins_before) + osk.new_time_windows(ps, pe), values_before=values)


def tie_service(n=6, cached=2):
    """Millisecond clocks, two parallel callees at fixed offsets from the in-span's start, and every span
    of a callee ending at one common instant (so the parent search of BuildDistributions samples the
    same tail for every in-span); trace `cached` has its callee-1 call cached.  Every delay law is then
    a single value: the in-span's own full tuple and its tuple with the skip span (incoming -> callee 0
    -> back) both score exactly the density at the mean, and the reference, comparing a skip span with
    a real span, raises."""
    in_s = synth.T0 + np.arange(n, dtype=np.int64) * 10_000
    end = synth.T0 + n * 10_000 + 20_000
    in_e = np.full(n, end + 2000, np.int64)
    keep = np.arange(n) != cached
    out_s = [in_s + 1000, (in_s + 3000)[keep]]
    out_e = [np.full(n, end - 1000, np.int64), np.full(int(keep.sum()), end, np.int64)]
    truth = np.stack([np.arange(n), np.where(keep, np.cumsum(keep) - 1, -2)]).astype(np.int32)
    return SkipService(name=f"tie-skip-real-n{n}-cached{cached}", in_start=in_s, in_end=in_e, out_start=out_s,
                       out_end=out_e, preds=[[], []], truth=truth)


def _variants(shape):
    E = len(DAG8["preds"]) if shape == "dag8" else len(synth.SHAPES[shape]["preds"])
    n = 120 if shape == "dag8" else 200
    load = dict(dag8=60.0).get(shape, 20.0 if shape.startswith("ali") else 60.0 if shape.startswith("media") else 100.0)
    mid = min(1, E - 1)
    return [
        # a cached callee in the middle of the DAG, microsecond clocks (E = 1: at the root, all-skip leaves)
        dict(shape=shape, n=n, load=load, seed=11, cached=(mid,), rate=0.2, quantum=1),
        # millisecond clocks: the root cached and more calls than in-spans on the last callee (mixed signs)
        dict(shape=shape, n=n, load=load, seed=12, cached=(0,) if E > 1 else (), rate=0.2, quantum=1000,
             extra=((E - 1, 10),)),
        # no cache hit, more calls than in-spans: no positive budget, log-density sums
        dict(shape=shape, n=n, load=load, seed=13, quantum=1000, extra=((0, 12),)),
    ]


def matrix():
    """The generated services of the skip tests: (id, builder).  Builders are cheap; ids name the input."""
    specs = [v for shape in SHAPES + ["dag8"] for v in _variants(shape)]
    specs += [   # every callee but the last cached: chains of skipped ancestors / all-skip tuples
        dict(shape="hotel_frontend", n=200, load=100.0, seed=21, cached=(0, 1), rate=0.2, quantum=1000),
        dict(shape="ali_chain4", n=200, load=20.0, seed=22, cached=(1, 2), rate=0.2, quantum=1000),
        dict(shape="media_nginx", n=200, load=60.0, seed=23, cached=(0, 1, 2, 3), rate=0.2),
        dict(shape="dag8", n=120, load=60.0, seed=24, cached=(1, 5), rate=0.2),
        dict(shape="ali_chain4", n=200, load=20.0, seed=25, cached=(1,), rate=0.3, quantum=1000, extra=((3, 5),)),
        # the last callee cached: earlier (parallel) callees shift and arrive out of order, and the order in
        # which the with-deletion search visits them decides which skip span each tuple fetches
        dict(shape="media_nginx", n=200, load=100.0, seed=26, cached=(3,), rate=0.3),
        dict(shape="media_nginx_cal", n=200, load=60.0, seed=27, cached=(3,), rate=0.3, quantum=1000),
        dict(shape="ali_par3", n=200, load=60.0, seed=27, cached=(2,), rate=0.3),
        dict(shape="dag8", n=120, load=60.0, seed=29, cached=(6,), rate=0.3),
    ]
    out = []
    for s in specs:
        kw = {k: v for k, v in s.items() if k != "shape"}
        out.append((make_service(s["shape"], **kw).name, lambda s=s, kw=kw: make_service(s["shape"], **kw)))
    for shape, cached, q in (("hotel_frontend", (1,), 1000), ("media_nginx", (2,), 1), ("dag8", (2,), 1000)):
        n = 120 if shape == "dag8" else 200
        load = 60.0 if shape != "hotel_frontend" else 100.0

        def build(shape=shape, cached=cached, q=q, n=n, load=load):
            svc = make_service(shape, n=n, load=load, seed=31, cached=cached, rate=0.2, quantum=q)
            prior = make_service(shape, n=n, load=load, seed=32, cached=cached, rate=0.1, quantum=q)
            return with_history(svc, prior)
        out.append((build().name, build))
    for shape, cached in (("hotel_frontend", (1,)), ("media_nginx", (2,))):
        # the same service twice through one instance: every window appears twice with one start, and
        # the in-spans must fetch from the first of each pair (its skip spans have the lower numbers)
        def build(shape=shape, cached=cached):
            svc = make_service(shape, n=200, load=100.0, seed=33, cached=cached, rate=0.2)
            return with_history(svc, svc)
        out.append((build().name, build))
    out.append((tie_service().name, tie_service))
    return out


K = _abi.TW_K
RTOL = 1e-12      # device exp() / log() against NumPy's (test_skip_mode)


def assert_equals_oracle(res, ref):
    """A result of the engine's search (skipmode.solve or the stepped device code: caller's positions)
    against solve_skip's: indices, counts and windows exactly, scores to RTOL, the counters."""
    from oracle import tw_oracle
    assert tw_oracle.windows_from_cuts(res["cut"]) == [tuple(w) for w in ref["windows"]]
    for mine, theirs in (("assign", "assign"), ("mis_rank", "mis_rank"), ("n_cand", "n_cand"),
                         ("topk_idx", "topk_idx"), ("topk_cnt", "topk_cnt"), ("top2_idx", "topk2_idx"),
                         ("top2_cnt", "topk2_cnt")):
        assert np.array_equal(np.asarray(res[mine]).reshape(np.shape(ref[theirs])), ref[theirs]), mine
    for mine, theirs in (("topk_score", "topk_score"), ("top2_score", "topk2_score")):
        assert np.allclose(res[mine], ref[theirs], rtol=RTOL, atol=0, equal_nan=True), mine
    assert int(res["counters"][0, 0]) == ref["not_best_count"]
    assert int(res["counters"][0, 1]) == ref["cnt_unassigned"]
