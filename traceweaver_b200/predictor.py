"""Drop-in predictor: the reference's plugin interface for the accelerated path.

Mirrors `TraceWeaverV3` of the reference (src/trace_reconstructor/ports/python/algorithms/
traceweaver_v3.py:29, constructed as `Cls(all_spans, all_processes)` and registered in
executor.py:888-900) for method "MaxScoreBatchSubsetWithSkips": same constructor, same
`FindAssignments` signature (traceweaver_v3.py:1087), same 6-tuple result (:1229), so the
reference's executor.py and helpers/utils.py accuracy code run unmodified on top of it (see
INTEGRATION.md).  All compute is in the CUDA engine behind the C ABI; this file only marshals
`Span` objects to SoA arrays and index results back to span ids.
"""
import numpy as np

from . import _abi, refit, skipmode
from .batch import Problem, build_batch
from .engine import Engine, _to_device

METHOD = "MaxScoreBatchSubsetWithSkips"
NA = ("NA", "NA")
SKIP = ("Skip", "Skip")


def solve_batch(eng: Engine, hb, seed_select=10, truth_assign=None, term_order=None, device_arrays=None,
                pinned=False, keep=("assign", "mis_rank", "counters", "n_cand", "topk"), want_likelihood=False):
    """The whole path for a bound-able batch: both passes of traceweaver_v3.py:1159-1227.

    params0 -> windows -> stitch (pass 0) -> delays -> refit -> score (final top-K) -> stitch
    (pass 1).  Returns device tensors; one host sync at the end (engine status)."""
    eng.bind(hb, device_arrays=device_arrays, pinned=pinned)
    return solve_bound(eng, seed_select, truth_assign, term_order, want_likelihood=want_likelihood)


def solve_bound(eng: Engine, seed_select=10, truth_assign=None, term_order=None, check=True, after_score=None,
                want_likelihood=False):
    """Both passes over the batch currently bound to `eng` (inputs resident in HBM).  check=False
    leaves the one host sync (engine status) to the caller, who must call eng.status().
    `after_score(top)` is called as soon as the final top-K lists are queued (before the last
    stitch), so a caller can start copying them out while the stitch runs.
    want_likelihood: also score the final assignment under the refitted mixtures against the final
    top-K (Engine.score_assignments): result["likelihood"]."""
    eng.prepare()                                 # prev-index scan, sorted end times
    p0 = eng.params_pass0()                       # ComputeEpPairDistParams3, every 100-span batch
    # CreateWindows2 (perfect-cut flags) + FindTopKAssignments on the undeleted lists, pass-0 params
    sc = eng.score(p0, want_used=True)
    r0 = eng.stitch(p0, sc["cut"], undeleted=sc)  # iteration 0
    delays, counts = eng.delays(r0["assign"])     # ComputeEpPairDistParams5: durations
    base = None
    if truth_assign is not None:
        # the reference fits (and discards) GMMs on the TRUE assignments first; they only advance
        # NumPy's global random stream (SURVEY A.9 item 7)
        dt, ct = eng.delays(truth_assign)
        base = eng.gmm_stream_draws(dt, ct)
    p1 = eng.gmm_refit(delays, counts, seed_select=seed_select, prob_base_skip=base, term_order=term_order)
    # top_k_2 of the last iteration -> all_topk_assignments; candidate maps are parameter independent
    top = eng.score(p1, out=dict(used_lo=sc["used_lo"], used_bits=sc["used_bits"], used_wide=sc["used_wide"],
                                 cut=sc["cut"]), keep_windows=True)
    if after_score is not None:
        after_score(top)
    r1 = eng.stitch(p1, sc["cut"], undeleted=top)  # iteration 1
    # the status column: a service that hit a search limit in either pass (counters[p, 3] < 0 and the
    # engine's error flag; the last pass alone would hide a first-pass failure)
    r1["counters"][:, 3] = r1["counters"][:, 3].minimum(r0["counters"][:, 3])
    n_cand = r0["n_cand"] + r1["n_cand"]          # per_span_candidates accumulates over iterations
    lik = eng.score_assignments(p1, r1["assign"], final_topk=top) if want_likelihood else None
    if check:
        eng.status()
    res = dict(assign=r1["assign"], mis_rank=r1["mis_rank"], counters=r1["counters"], n_cand=n_cand,
               topk_score=top["topk_score"], topk_idx=top["topk_idx"], topk_cnt=top["topk_cnt"],
               cut=sc["cut"], params_pass1=p1, assign_pass0=r0["assign"])
    if want_likelihood:
        res["likelihood"] = lik
    return res


class TraceWeaverV3:
    """`predictors` entry replacing the reference's ("MaxScoreBatchSubsetWithSkips", TraceWeaverV3).

    want_likelihood=True: every FindAssignments call also scores its own final assignment under the model
    it solved with and leaves `self.last_likelihood`:
        in_spans       {in-span id: (score, code, margin)}   code TW_ASSESS_* (1 = unassigned), score NaN
                       unless code 0, margin s0 - s1 (+inf) when the chosen tuple is the best one, else score - s0
        service_score  sum of the scored in-spans' scores
        service_codes  in-spans per code
        regime         "two_pass": scores are log-likelihoods under the refitted mixtures;
                       "skip" (a service with skip budgets): the skip regime's scores, means of densities
                       where a budget is positive, so the two are not comparable
    The 6-tuple is the same either way."""

    def __init__(self, all_spans, all_processes, device=0, seed_select=10, carry_state=True, want_likelihood=False):
        self.all_spans = all_spans
        self.all_processes = all_processes
        self.seed_select = seed_select
        self.engine = Engine(device)          # raises without a CUDA device: there is no CPU path
        self.last = None
        self.want_likelihood = want_likelihood
        self.last_likelihood = None
        # what the reference's instance keeps from one service to the next and its skip regime reads
        # (time_windows, distribution_values: traceweaver_v3.py:40,45 are never reset)
        self.skip_state = skipmode.SkipState()
        self.carry_state = carry_state
        self._pending_dist = []
        self._fractional_state = False        # parked skip-regime state came from a service with float times

    # -- marshalling -------------------------------------------------------------------------------
    @staticmethod
    def _fractional(spans):
        return any(isinstance(sp.start_mus, float) and sp.start_mus != int(sp.start_mus) for sp in spans)

    @staticmethod
    def _arrays(spans, fractional=False):
        """(start, end) arrays.  fractional: float64 microseconds — executor.py --compress_factor > 1
        (transforms.repeat_change_spans) divides the start times — with end = start_mus + duration_mus
        formed in Python float arithmetic as the reference does; the engine solves them in exact fixed
        point (tw_engine_bind_f64)."""
        if fractional:
            s = np.fromiter((float(sp.start_mus) for sp in spans), np.float64, len(spans))
            e = np.fromiter((float(sp.start_mus) + sp.duration_mus for sp in spans), np.float64, len(spans))
            return s, e
        s = np.fromiter((int(sp.start_mus) for sp in spans), np.int64, len(spans))
        d = np.fromiter((sp.duration_mus for sp in spans), np.int64, len(spans))
        return s, s + d

    def _marshal(self, process, in_spans, partitions, invocation_graph, fractional):
        """The Problem of one service solved on `partitions` (the outgoing lists in the order the regime
        solves them on), the topological callee order and the span ids (in_ids, out_ids per callee)."""
        import networkx as nx
        out_eps = list(nx.topological_sort(invocation_graph))            # traceweaver_v1.py:37-39
        if set(out_eps) != set(partitions.keys()):
            raise ValueError("invocation_graph nodes must be the outgoing endpoints")
        pos = {ep: i for i, ep in enumerate(out_eps)}
        in_s, in_e = self._arrays(in_spans, fractional)
        outs = [self._arrays(partitions[ep], fractional) for ep in out_eps]
        preds = [[pos[b] for b, _ in invocation_graph.in_edges(ep)] for ep in out_eps]
        prob = Problem(in_start=in_s, in_end=in_e, out_start=[o[0] for o in outs], out_end=[o[1] for o in outs],
                       preds=preds, name=process)
        in_ids = [s.GetId() for s in in_spans]
        out_ids = [[s.GetId() for s in partitions[ep]] for ep in out_eps]
        return prob, out_eps, in_ids, out_ids

    @staticmethod
    def _result(in_ids, out_eps, out_ids, assign, topk_idx, topk_cnt, n_cand, counters, given_eps,
                true_assignments):
        """The reference's 6-tuple (traceweaver_v3.py:1229) from index results: assign [E, n] and
        topk_idx [n, K, E] hold positions in the lists of `out_ids`, -1 for ("NA", "NA") and, in the
        skip regime only, <= -2 for ("Skip", "Skip") (traceweaver_v1.py:446-453)."""
        n = len(in_ids)

        def name(e, c):
            return out_ids[e][c] if c >= 0 else (NA if c == -1 else SKIP)
        all_assignments = {ep: {in_ids[i]: name(e, int(assign[e, i])) for i in range(n)} for e, ep in enumerate(out_eps)}
        all_topk = {ep: {in_ids[i]: [name(e, int(topk_idx[i, r, e])) for r in range(topk_cnt[i])] for i in range(n)}
                    for e, ep in enumerate(out_eps)}
        per_span_candidates = {}
        for ep in given_eps:                                             # traceweaver_v3.py:1096-1098
            for key in (true_assignments.get(ep, {}) if true_assignments else {}):
                per_span_candidates[key] = 0
        for i in range(n):
            if n_cand[i] or in_ids[i] in per_span_candidates:
                per_span_candidates[in_ids[i]] = int(n_cand[i])
        return (all_assignments, all_topk, int(counters[0, 0]), n, per_span_candidates, int(counters[0, 1]))

    @staticmethod
    def _likelihood(regime, in_ids, score, code, margin, service_score, service_codes):
        return dict(in_spans={iid: (float(score[i]), int(code[i]), float(margin[i])) for i, iid in enumerate(in_ids)},
                    service_score=float(service_score), service_codes=np.asarray(service_codes), regime=regime)

    # -- the reference's entry point ---------------------------------------------------------------
    def FindAssignments(self, method, process, in_span_partitions, out_span_partitions, parallel,
                        instrumented_hops, true_assignments, invocation_graph, true_skips=False,
                        true_dist=False):
        assert len(in_span_partitions) == 1                              # traceweaver_v3.py:1088
        if method != METHOD or true_skips or true_dist:
            raise NotImplementedError(
                f"traceweaver_b200 accelerates method {METHOD!r} only (got {method!r}); the ablation "
                "variants stay with the reference implementation")
        in_ep, in_spans = list(in_span_partitions.items())[0]
        # TallySkipSpans re-sorts every partition by start (stable), traceweaver_v3.py:968-971
        in_spans = sorted(in_spans, key=lambda x: float(x.start_mus))
        frac = self._fractional(in_spans) or any(self._fractional(p) for p in out_span_partitions.values())
        if any(len(p) != len(in_spans) for p in out_span_partitions.values()):
            # skip budgets (cache hits / dynamism): ONE iteration with skip spans, traceweaver_v3.py:1138-1158
            if frac:
                raise NotImplementedError("fractional start_mus (time-compressed spans) on a service with skip "
                                          "budgets: the skip regime keeps int64 timestamps; use the reference")
            if self.carry_state and self._fractional_state:
                raise NotImplementedError("a service with skip budgets after a service with fractional start_mus: "
                                          "the skip regime would read state built from fractional timestamps; "
                                          "use carry_state=False or the reference")
            # the caller's list order: skipmode.solve sorts the lists itself and names results in this order
            prob, out_eps, in_ids, out_ids = self._marshal(process, in_spans, out_span_partitions, invocation_graph,
                                                           frac)
            state = self.skip_state if self.carry_state else skipmode.SkipState()
            for a in self._pending_dist:              # BuildDistributions of the earlier services, in call order
                skipmode.build_distributions(self.engine, *a[:4], a[4], state)
            self._pending_dist = []
            res = skipmode.solve(self.engine, prob.in_start, prob.in_end, prob.out_start, prob.out_end, prob.preds,
                                 labels=[in_ep] + out_eps, state=state, want_topk=False,
                                 want_likelihood=self.want_likelihood)
            self.last = res
            if self.want_likelihood:
                self.last_likelihood = self._likelihood("skip", in_ids, res["chosen_score"], res["chosen_code"],
                                                        res["margin"], res["service_score"], res["service_codes"])
            return self._result(in_ids, out_eps, out_ids, res["assign"], res["top2_idx"], res["top2_cnt"],
                                res["n_cand"], res["counters"], out_span_partitions.keys(), true_assignments)
        out_parts = {ep: sorted(p, key=lambda x: float(x.start_mus)) for ep, p in out_span_partitions.items()}
        prob, out_eps, in_ids, out_ids = self._marshal(process, in_spans, out_parts, invocation_graph, frac)
        hb = build_batch([prob])
        n, E = prob.n_in, prob.E
        # ground truth only advances the refit's random stream, exactly as in the reference
        truth = np.full((E, n), -1, np.int32)
        for e, ep in enumerate(out_eps):
            lut = {sid: j for j, sid in enumerate(out_ids[e])}
            ta = true_assignments.get(ep, {}) if true_assignments else {}
            truth[e] = [lut.get(ta.get(i), -1) for i in in_ids]
        given_pos = [out_eps.index(ep) for ep in out_span_partitions.keys()]
        order = np.asarray(refit.reference_term_order(prob, given_pos), np.int32)

        if self.carry_state:
            # the reference runs TallySkipSpans and BuildDistributions for EVERY service (v3:1136, :1149);
            # in this regime they only leave state behind for a later service with skip budgets: the time
            # windows are appended now (a few tuples), the distribution samples are derived lazily — the
            # arrays are parked and run through tw_build_dist_samples, in call order, when a service with
            # skip budgets actually arrives
            self._fractional_state |= hb.float_times
            self.skip_state.time_windows.extend(skipmode.new_time_windows(prob.in_start, prob.in_end))
            self._pending_dist.append((prob.in_start, prob.in_end, prob.out_start, prob.out_end, [in_ep] + out_eps))
        res = solve_batch(self.engine, hb, seed_select=self.seed_select, want_likelihood=self.want_likelihood,
                          **_to_device(dict(truth_assign=truth.reshape(-1), term_order=order), self.engine.device))
        self.last = res
        if self.want_likelihood:
            lk = {k: v.cpu().numpy() for k, v in res["likelihood"].items()}
            self.last_likelihood = self._likelihood("two_pass", in_ids, lk["score"], lk["code"], lk["margin"],
                                                    lk["prob_sum"][0], lk["prob_count"][0])
        host = {k: res[k].cpu().numpy() for k in ("assign", "topk_idx", "topk_cnt", "n_cand", "counters")}
        return self._result(in_ids, out_eps, out_ids, host["assign"].reshape(E, n),
                            host["topk_idx"].reshape(n, _abi.TW_K, E), host["topk_cnt"], host["n_cand"],
                            host["counters"], out_span_partitions.keys(), true_assignments)
