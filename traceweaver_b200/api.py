"""Public batch API: many services per call, HOST buffers in, HOST buffers out.

    solver = BatchSolver(device=0)
    out = solver.solve(host_batch)        # HostBatch from batch.build_batch / build_batch_from_blocks
    out["assign"]   int32  [sum n_in*E]   assign[tuple_off[p] + e*n_in_p + i] -> index in ep e's list, -1 = NA
    out["topk_idx"] int32  [5*sum n_in*E] final no-deletion top-K tuples (all_topk_assignments)
    out["topk_cnt"] uint8  [sum n_in]
    out["n_cand"]   int32  [sum n_in]     per_span_candidates (both iterations)
    out["counters"] int32  [P, 4]         not_best_count, cnt_unassigned, max MWIS nodes, status

This is `TraceWeaverV3.FindAssignments` (traceweaver_v3.py:1087-1229) for every service of the
batch in one launch sequence; `predictor.TraceWeaverV3` is the same path behind the reference's
one-service-at-a-time plugin signature.  Every call copies the caller's span arrays into page-locked
staging buffers (a host memcpy, every call: the caller may refill its buffers in place), sends them
host->device, and brings the results device->host; nothing about the batch CONTENTS is cached across
calls — only buffers (device scratch, staging, result buffers) are re-used.

Result lifetime: the returned arrays are views of page-locked result buffers owned by the solver.
Two sets alternate, so the arrays of a call stay valid until the SECOND next call of `solve()`;
copy them if you keep them longer (`np.array(out["assign"])`).
"""
import numpy as np
import torch

from . import _abi
from .batch import HostBatch
from .engine import Engine, _to_device
from .predictor import solve_bound


class BatchSolver:
    """`chunks` > 1 splits the services of a batch into that many groups and runs them round-robin on
    two CUDA streams (one engine each), so that a group's host->device and device->host copies
    overlap another group's kernels.  The groups are independent problems: results are identical.
    Four groups measured best on the 8192-service bench workload (H100 SXM 80 GB at a 700 W limit,
    median of four alternating rounds of ten calls: 74.7 ms in two groups, 73.2 in three, 71.2 in four;
    scripts/time_e2e.py compares group counts)."""

    #: below this many in-spans a batch is solved in one piece (copies are not worth hiding)
    MIN_CHUNK_IN_SPANS = 1 << 20
    #: share of the in-spans in the first of two groups
    FIRST_GROUP_FRACTION = 0.5

    def __init__(self, device=0, seed_select=10, chunks=4):
        self.engine = Engine(device)
        self.seed_select = seed_select
        self.chunks = max(1, int(chunks))
        self._engines = [self.engine]
        self._streams = None
        self._copy_stream = None
        self._pinned_in = {}
        self._pinned_out = [{}, {}]
        self._flip = 0
        self.last_chunks = 1
        self.h2d_bytes = 0
        self.d2h_bytes = 0

    def close(self):
        for e in self._engines:
            e.close()

    def _stage(self, name, a):
        """Copy the caller's host array into a page-locked staging buffer (allocated once per
        shape; the copy happens on EVERY call — the buffer's address says nothing about its contents)."""
        src = a.view(np.int32) if a.dtype == np.uint32 else a
        src = torch.from_numpy(np.ascontiguousarray(src))
        t = self._pinned_in.get(name)
        if t is None or t.shape != src.shape or t.dtype != src.dtype:
            t = torch.empty(src.shape, dtype=src.dtype, pin_memory=True)
            self._pinned_in[name] = t
        t.copy_(src)
        return t

    def _out_buf(self, name, n, dtype, cols=None):
        shape = (n,) if cols is None else (n, cols)
        bufs = self._pinned_out[self._flip]
        buf = bufs.get(name)
        if buf is None or tuple(buf.shape) != shape or buf.dtype != dtype:
            buf = torch.empty(shape, dtype=dtype, pin_memory=True)
            bufs[name] = buf
        return buf

    def _chunk_plan(self, hb: HostBatch):
        """[(lo, hi, sub-batch)]: recomputed every call (O(P) descriptor arithmetic, span arrays are views)."""
        n_in = int(hb.prob_in_off[-1])
        C = self.chunks if n_in >= self.MIN_CHUNK_IN_SPANS else 1
        C = min(C, hb.n_problems)
        if C == 1:
            return [(0, hb.n_problems, hb)]
        # a first group (its host->device copy is the only one nothing can hide), the rest in equal
        # in-span counts
        first = self.FIRST_GROUP_FRACTION if (C == 2 or self.FIRST_GROUP_FRACTION < 1.0 / C) else 1.0 / C
        fr = first + (1.0 - first) * np.arange(0, C - 1) / max(C - 1, 1)
        cuts = np.searchsorted(hb.prob_in_off, fr * n_in, side="left")
        edges = sorted(set([0, hb.n_problems] + [int(c) for c in cuts if 0 < c < hb.n_problems]))
        return [(lo, hi, hb.slice(lo, hi)) for lo, hi in zip(edges[:-1], edges[1:])]

    def solve(self, hb: HostBatch, truth_assign=None, term_order=None, want_scores=False, strict=True,
              want_likelihood=False, want_mixtures=False):
        """want_scores: also return out["topk_score"] (float64 [sum n_in, 5]; the reference's 6-tuple
        carries the top-K ids only, traceweaver_v3.py:1229, so the scores stay on the device by default).

        want_likelihood: how confident each choice is.  The final assignment is scored under the refitted
        mixtures (tw_score_assignments) and compared with the final top-K:
            out["chosen_score"]   float64 [sum n_in]  log-likelihood of the chosen tuple, NaN if not scored
            out["chosen_code"]    uint8   [sum n_in]  TW_ASSESS_* (0 scored, 1 unassigned, ...)
            out["margin"]         float64 [sum n_in]  chosen = rank 0: s0 - s1 (+inf: single candidate),
                                                      else score - s0 (<= 0); NaN if not scored
            out["service_loglik"] float64 [P]         sum of the scored in-spans' log-likelihoods
            out["service_codes"]  int32   [P, 5]      in-spans per code
        want_mixtures: out["mixtures"] float64 [n_terms, TW_MIX_REC], the refitted delay model (term order of
        the batch), and out["mixture_off"] int64 [P+1], the first term of every service; score() takes them.

        strict=False: a service that runs into a search limit of the engine (TW_ERR_MWIS_LIMIT: more
        than 2 M branch-and-bound nodes in one window) no longer fails the whole call: the other
        services' results are returned, out["counters"][p, 3] holds the status of service p (0 = ok;
        the in-spans of a failed service after the failing window stay unassigned) and
        out["failed_services"] lists the failed ones.  Anything else still raises."""
        dev = self.engine.device
        self._flip ^= 1
        single = truth_assign is not None or term_order is not None
        plan = [(0, hb.n_problems, hb)] if single else self._chunk_plan(hb)
        if len(plan) > 1 and self._streams is None:
            self._engines.append(Engine(dev.index if dev.index is not None else 0))
            self._streams = [torch.cuda.Stream(dev), torch.cuda.Stream(dev)]
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(dev)
        n_in, n_tuple = int(hb.prob_in_off[-1]), int(hb.prob_tuple_off[-1])
        out = dict(
            assign=self._out_buf("assign", n_tuple, torch.int32),
            topk_idx=self._out_buf("topk_idx", _abi.TW_K * n_tuple, torch.int32),
            topk_cnt=self._out_buf("topk_cnt", n_in, torch.uint8),
            n_cand=self._out_buf("n_cand", n_in, torch.int32),
            counters=self._out_buf("counters", hb.n_problems, torch.int32, 4),
            mis_rank=self._out_buf("mis_rank", n_in, torch.int8))
        if want_scores:
            out["topk_score"] = self._out_buf("topk_score", n_in, torch.float64, _abi.TW_K)
        if want_likelihood:
            out.update(chosen_score=self._out_buf("chosen_score", n_in, torch.float64),
                       chosen_code=self._out_buf("chosen_code", n_in, torch.uint8),
                       margin=self._out_buf("margin", n_in, torch.float64),
                       service_loglik=self._out_buf("service_loglik", hb.n_problems, torch.float64),
                       service_codes=self._out_buf("service_codes", hb.n_problems, torch.int32, _abi.TW_ASSESS_NCODES))
        mixture_off = hb.ep_term_off[hb.prob_ep_off].astype(np.int64)
        if want_mixtures:
            out["mixtures"] = self._out_buf("mixtures", int(mixture_off[-1]), torch.float64, _abi.TW_MIX_REC)
        self.last_chunks = len(plan)
        h2d = d2h = 0
        main = torch.cuda.current_stream(dev)
        used = []
        for c, (lo, hi, sub) in enumerate(plan):
            eng = self._engines[c % len(self._engines)] if len(plan) > 1 else self.engine
            stream = self._streams[c % 2] if len(plan) > 1 else main
            if len(plan) > 1 and c < 2:
                stream.wait_stream(main)
            with torch.cuda.stream(stream):
                d = {}
                for name, a in sub.arrays.items():
                    p = self._stage((c, name), a)
                    d[name] = p.to(dev, non_blocking=True)        # H2D inside the caller's timed region
                    h2d += p.numel() * p.element_size()
                eng.bind(sub, device_arrays=d)
                inputs = _to_device({k: None if v is None else np.asarray(v, np.int32)
                                     for k, v in (("truth_assign", truth_assign), ("term_order", term_order))}, dev)
                i0, t0 = int(hb.prob_in_off[lo]), int(hb.prob_tuple_off[lo])
                i1, t1 = int(hb.prob_in_off[hi]), int(hb.prob_tuple_off[hi])

                def copy_topk(top, stream=stream, i0=i0, i1=i1, t0=t0, t1=t1):
                    # the top-K lists (three quarters of the result bytes) are final before the last
                    # stitch: copy them out on the copy stream while that kernel runs
                    ev = torch.cuda.Event()
                    ev.record(stream)
                    self._copy_stream.wait_event(ev)
                    with torch.cuda.stream(self._copy_stream):
                        names = [("topk_idx", (_abi.TW_K * t0, _abi.TW_K * t1)), ("topk_cnt", (i0, i1))]
                        if want_scores:
                            names.append(("topk_score", (i0, i1)))
                        for name, (b0, b1) in names:
                            t = top[name]
                            t.record_stream(self._copy_stream)
                            out[name][b0:b1].copy_(t, non_blocking=True)

                res = solve_bound(eng, seed_select=self.seed_select, check=False, after_score=copy_topk,
                                  want_likelihood=want_likelihood, **inputs)
                d2h += sum(res[k].numel() * res[k].element_size()
                           for k in ("topk_idx", "topk_cnt") + (("topk_score",) if want_scores else ()))
                for name, (b0, b1) in (("assign", (t0, t1)), ("n_cand", (i0, i1)), ("counters", (lo, hi)),
                                       ("mis_rank", (i0, i1))):
                    t = res[name]
                    out[name][b0:b1].copy_(t, non_blocking=True)  # D2H
                    d2h += t.numel() * t.element_size()
                extra = []
                if want_likelihood:
                    lk = res["likelihood"]
                    extra += [("chosen_score", lk["score"], i0, i1), ("chosen_code", lk["code"], i0, i1),
                              ("margin", lk["margin"], i0, i1), ("service_loglik", lk["prob_sum"], lo, hi),
                              ("service_codes", lk["prob_count"], lo, hi)]
                if want_mixtures:
                    extra.append(("mixtures", res["params_pass1"].table, int(mixture_off[lo]), int(mixture_off[hi])))
                if extra:                                         # D2H on the copy stream, as the top-K lists
                    ev = torch.cuda.Event()
                    ev.record(stream)
                    self._copy_stream.wait_event(ev)
                    with torch.cuda.stream(self._copy_stream):
                        for name, t, b0, b1 in extra:
                            t.record_stream(self._copy_stream)
                            out[name][b0:b1].copy_(t, non_blocking=True)
                            d2h += t.numel() * t.element_size()
            used.append((eng, stream))
        self._copy_stream.synchronize()
        limit_hit = False
        for eng, stream in dict((id(e), (e, s)) for e, s in used).values():
            with torch.cuda.stream(stream):
                try:
                    eng.status()                                  # syncs the stream, raises on engine errors
                except _abi.TwError as ex:
                    if strict or ex.code != _abi.TW_ERR_MWIS_LIMIT:
                        raise
                    limit_hit = True
            main.wait_stream(stream)
        self.h2d_bytes, self.d2h_bytes = h2d, d2h
        res = {k: v.numpy() for k, v in out.items()}
        if want_mixtures:
            res["mixture_off"] = mixture_off
        if not strict:
            res["failed_services"] = np.flatnonzero(res["counters"][:, 3] != 0) if limit_hit else np.zeros(0, np.int64)
        return res

    def score(self, hb: HostBatch, assign, mixtures):
        """The likelihood of ANY assignment of `hb` (the layout of out["assign"]: an earlier result, the
        loader's ground truth, another predictor's answer) under mixtures an earlier
        solve(hb, want_mixtures=True) returned.  Host arrays: score / code [sum n_in] (code TW_ASSESS_*,
        score NaN unless code 0), service_loglik [P], service_codes [P, TW_ASSESS_NCODES]."""
        n_tuple, n_terms = int(hb.prob_tuple_off[-1]), int(hb.ep_term_off[-1])
        assign = np.asarray(assign, np.int32).reshape(-1)
        mixtures = np.asarray(mixtures, np.float64)
        if assign.shape != (n_tuple,) or mixtures.shape != (n_terms, _abi.TW_MIX_REC):
            raise ValueError(f"score: assign must have {n_tuple} entries and mixtures shape ({n_terms}, "
                             f"{_abi.TW_MIX_REC}) for this batch")
        eng = self.engine
        eng.bind(hb)
        prm = eng.params_from_host(mix=mixtures)
        lk = eng.score_assignments(prm, _to_device(dict(assign=assign), eng.device)["assign"])
        eng.status()
        return dict(score=lk["score"].cpu().numpy(), code=lk["code"].cpu().numpy(),
                    service_loglik=lk["prob_sum"].cpu().numpy(), service_codes=lk["prob_count"].cpu().numpy())

    def assemble(self, hb: HostBatch, assign, in_caller, truth=None):
        """End-to-end request trees of the whole batch `hb` (tw_assemble_traces; whatever grouping solve()
        used): `assign` in the layout of out["assign"], `in_caller` from traces.caller_links.  Host arrays
        over the nodes (in-span g is node g, out-span j node n_in + j): parent, root (-1 on or under a cycle),
        size (nodes per root).  With `truth` (an assignment in the same layout, e.g. the loader's ground
        truth) also exact [n_in], int8: for an in-span root r, 1 iff the request rooted at r holds exactly the
        nodes it holds under the truth; -1 for an in-span that is not a root."""
        from . import traces
        eng = self.engine
        links = traces.upload_inputs(eng, hb, "assemble", in_caller=in_caller)["in_caller"]
        res = traces.assemble(eng, hb, assign, links)
        out = {k: v.cpu().numpy() for k, v in res.items()}
        if truth is not None:
            ref = traces.assemble(eng, hb, truth, links)
            out["exact"] = traces.exact_requests(res["root"], ref["root"], int(hb.prob_in_off[-1])).cpu().numpy()
        return out

    def critical_paths(self, hb: HostBatch, assign, in_caller, slow_quantile=0.99):
        """Where the time of every reconstructed request of `hb` went (tw_critical_paths; definition in
        traces.py): `assign` in the layout of out["assign"], `in_caller` from traces.caller_links.  The slow
        requests are those whose latency is at least the lower `slow_quantile`-quantile of all request
        latencies (an actual latency, computed on the device).  Host arrays: root, on_path, self_us [nodes],
        culprit [n_in], server_us / server_visits [P, 2] and call_us [n_ep, 2] (column 0 all requests,
        column 1 slow ones), requests [2]; request (node ids of the request roots) and latency_us [requests];
        slow_us, the threshold."""
        from . import traces
        eng = self.engine
        spans = traces.upload_spans(eng, hb)
        links = traces.upload_inputs(eng, hb, "critical_paths", in_caller=in_caller)["in_caller"]
        req, lat = traces.request_latencies(spans, links)
        slow_us = traces.lower_quantile(lat, slow_quantile)
        res = traces.critical_paths(eng, hb, assign, links, slow_us, spans=spans)
        eng.status()                                      # syncs the stream, raises on engine errors
        out = {k: v.cpu().numpy() for k, v in res.items()}
        out.update(request=req.cpu().numpy(), latency_us=lat.cpu().numpy(), slow_us=slow_us)
        return out

    def request_confidence(self, hb: HostBatch, out, in_caller):
        """How sure the reconstruction of every request of `hb` is, without a ground truth
        (tw_request_confidence; definition in traces.py).  `out`: a solve(hb, want_likelihood=True,
        want_scores=True) result, or any dict with the same keys: assign, chosen_score, chosen_code (the chosen
        tuples' scores, e.g. from score()), topk_score, topk_idx, topk_cnt (the final no-deletion top-K).
        `in_caller` from traces.caller_links.  Host arrays: root [nodes]; p, ell, decisions, zero, log_conf
        (int64, units of 2^-32 nats), conf, weakest, weakest_p [n_in]; est_accuracy [P]; requests and
        expected_exact (scalars); request, the node ids of the request roots."""
        from . import traces
        need = {"chosen_score": "want_likelihood=True", "chosen_code": "want_likelihood=True",
                "topk_score": "want_scores=True", "topk_idx": "want_scores=True", "topk_cnt": "want_scores=True",
                "assign": "a solve() result"}
        missing = [k for k in need if k not in out or out[k] is None]
        if missing:
            how = sorted({need[k] for k in missing})
            raise ValueError(f"request_confidence: `out` lacks {', '.join(missing)}; call solve() with "
                             f"{' and '.join(how)}")
        eng = self.engine
        res = traces.request_confidence(eng, hb, out["assign"], in_caller, out["chosen_score"], out["chosen_code"],
                                        {k: out[k] for k in ("topk_score", "topk_idx", "topk_cnt")})
        host = {k: v.cpu().numpy() for k, v in res.items()}
        n_in = int(hb.prob_in_off[-1])
        host["requests"] = int(host["requests"][0])
        host["expected_exact"] = float(host["expected_exact"][0])
        host["request"] = np.flatnonzero(host["root"][:n_in] == np.arange(n_in)).astype(np.int32)
        return host
