"""Reconstruct a directory of Jaeger JSON traces end to end: loader -> batch engine -> accuracy.

    python scripts/reconstruct_traces.py <trace dir> [--layout hotel|media|node|alibaba] [--device 0] [--likelihood]
                                         [--traces FILE.npz]

Prints, per solved service, the assignment accuracy against the traces' own parent links
(the reference's AccuracyForService, helpers/utils.py:34-60) and the time of each stage — the same
numbers executor.py prints for `--predictor_indices 10`.  --likelihood adds, per service, the mean
log-likelihood of the chosen tuples under the refitted delay model, quantiles of the margin to the runner-up
(or to the best tuple, for an in-span that did not get its best), and for the wrong in-spans whether the
true tuple scores above the chosen one (a search error: the window's MWIS and deletion pushed it out),
below it (a model error), or is infeasible.  --traces joins the assignments into end-to-end request trees on
the device (BatchSolver.assemble) and writes them to FILE.npz: parent, root, size per node (in-span g is node
g, out-span j node n_in + j), exact per in-span (1 / 0 for a reconstructed request that is / is not exactly its
trace, -1 for an in-span that is not a root) and the node -> (trace id, span id) tables node_trace_id,
node_span_id; it prints the share of exact requests beside the end-to-end accuracy.  --critical-path
(BatchSolver.critical_paths; definition in traceweaver_b200/traces.py) prints, per service and per callee
edge, the share of the requests' critical time spent there, over all requests and over the slow ones (latency at
or above the --slow-quantile of all latencies), on the predicted assignment and on the truth, and the largest
difference between the two; the services the slow requests' culprits belong to; and the share of exact requests
per latency decile.  With --traces the file also holds on_path, self_us and culprit of the prediction.
--confidence (BatchSolver.request_confidence; definition in traceweaver_b200/traces.py) prints, per service, the
truth-free est_accuracy beside the measured accuracy and the share of in-spans the window's MWIS did not give
their best tuple (not_best_count / n_in); the batch's expected_exact beside the exact share of requests; the
requests by confidence bin against their exact flag; and with --critical-path the culprit services of the slow
requests, split into confident (conf >= 0.99) and unconfident ones.  With --traces the file also holds conf,
weakest and p."""
import argparse, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("directory")
ap.add_argument("--layout", default="hotel", choices=["hotel", "media", "node", "alibaba"])
ap.add_argument("--device", type=int, default=0)
ap.add_argument("--seed", type=int, default=10)
ap.add_argument("--likelihood", action="store_true", help="print per-service confidence and error classes")
ap.add_argument("--traces", default=None, metavar="FILE.npz", help="write the reconstructed request trees")
ap.add_argument("--critical-path", action="store_true", help="print where the requests' time went")
ap.add_argument("--confidence", action="store_true", help="print how sure each reconstruction is, without the truth")
ap.add_argument("--slow-quantile", type=float, default=0.99, help="latency quantile of the slow requests")
args = ap.parse_args()

from traceweaver_b200.api import BatchSolver
from traceweaver_b200.loader import load_jaeger_dir, to_host_batch, accuracy, end_to_end_accuracy

t0 = time.perf_counter()
from traceweaver_b200.engine import Engine
_eng = Engine(args.device)
services = load_jaeger_dir(args.directory, layout=args.layout, engine=_eng)    # truth + FindOrder on the device
_eng.close()
# services with n_out == n_in at every callee go through the two-pass batch path; a raw trace directory holds
# no others (skip budgets come from executor.py's cache transform, see traceweaver_b200.skipmode)
ok = [s for s in services if all(len(o) == s.problem.n_in for o in s.problem.out_start)]
t1 = time.perf_counter()
print(f"loaded {len(services)} services ({len(ok)} without skip budgets) in {t1 - t0:.2f} s")
hb = to_host_batch(ok)
solver = BatchSolver(device=args.device, seed_select=args.seed)
solver.solve(hb)                                   # warm-up: allocations, random streams
t2 = time.perf_counter()
out = solver.solve(hb, want_likelihood=args.likelihood or args.confidence, want_mixtures=args.likelihood,
                   want_scores=args.confidence)
t3 = time.perf_counter()
n_spans = sum(s.problem.n_in * (1 + s.problem.E) for s in ok)
print(f"solved {n_spans} spans in {1e3 * (t3 - t2):.2f} ms (host buffers in and out)")
if args.likelihood:
    truth_all = np.concatenate([s.truth.reshape(-1) for s in ok]).astype(np.int32)
    tr = solver.score(hb, truth_all, out["mixtures"])       # the ground truth under the same delay model
for p, s in enumerate(ok):
    a = out["assign"][int(hb.prob_tuple_off[p]):int(hb.prob_tuple_off[p + 1])]
    print(f"  {s.name:28s} n_in={s.problem.n_in:5d} E={s.problem.E}  accuracy {100 * accuracy(s, a):7.3f} %")
    if not args.likelihood:
        continue
    i0, i1 = int(hb.prob_in_off[p]), int(hb.prob_in_off[p + 1])
    n_scored = int(out["service_codes"][p, 0])
    mean = out["service_loglik"][p] / n_scored if n_scored else float("nan")
    m = out["margin"][i0:i1]
    q = np.nanquantile(np.where(np.isinf(m), np.nan, m), [0.05, 0.25, 0.5]) if np.isfinite(m).any() else [np.nan] * 3
    wrong = ~(a.reshape(s.truth.shape) == s.truth).all(axis=0)
    ts, tc, cs = tr["score"][i0:i1][wrong], tr["code"][i0:i1][wrong], out["chosen_score"][i0:i1][wrong]
    cs = np.where(np.isnan(cs), -np.inf, cs)              # left unassigned: any feasible truth was pushed out
    feas = tc == 0
    print(f"      mean loglik {mean:9.3f}  margin q05/q25/q50 {q[0]:8.3f} {q[1]:8.3f} {q[2]:8.3f}  "
          f"single-candidate {int(np.isinf(m).sum())}  wrong {int(wrong.sum())}: search error "
          f"{int((feas & (ts > cs)).sum())}, model error {int((feas & (ts <= cs)).sum())}, "
          f"truth infeasible {int((~feas).sum())}")
cp = None
if args.critical_path:
    from traceweaver_b200 import traces
    in_caller = traces.caller_links(ok, hb)
    truth_all = np.concatenate([s.truth.reshape(-1) for s in ok]).astype(np.int32)
    t4 = time.perf_counter()
    cp = solver.critical_paths(hb, np.array(out["assign"]), in_caller, slow_quantile=args.slow_quantile)
    t5 = time.perf_counter()
    cpt = solver.critical_paths(hb, truth_all, in_caller, slow_quantile=args.slow_quantile)
    names = [s.name for s in ok]
    ep_names = [f"{s.name} -> callee {e}" for s in ok for e in range(s.problem.E)]
    print(f"critical paths ({1e3 * (t5 - t4):.2f} ms): {int(cp['requests'][0])} requests, "
          f"{int(cp['requests'][1])} slow (latency >= {cp['slow_us']:.1f} us, quantile {args.slow_quantile})")
    share = lambda r, col: np.concatenate([r["server_us"][:, col], r["call_us"][:, col]]) / \
        max(r["server_us"][:, col].sum() + r["call_us"][:, col].sum(), 1e-300)
    rows = names + ep_names
    pred = np.stack([share(cp, 0), share(cp, 1)], axis=1)
    true = np.stack([share(cpt, 0), share(cpt, 1)], axis=1)
    print(f"  {'service / callee edge':40s} {'all: pred':>10s} {'truth':>8s} {'slow: pred':>11s} {'truth':>8s}")
    for k, name in enumerate(rows):
        print(f"  {name:40s} {100 * pred[k, 0]:9.2f}% {100 * true[k, 0]:7.2f}% {100 * pred[k, 1]:10.2f}% "
              f"{100 * true[k, 1]:7.2f}%")
    diff = np.abs(pred - true)
    k, col = np.unravel_index(int(np.argmax(diff)), diff.shape)
    print(f"  largest difference: {100 * diff[k, col]:.2f} points at {rows[k]} ({('all', 'slow')[col]} requests)")
    n_in = int(hb.prob_in_off[-1])
    req = cp["request"]
    slow_req = req[cp["latency_us"] >= cp["slow_us"]]
    cul = cp["culprit"][slow_req]
    in_prob = np.repeat(np.arange(len(ok)), np.diff(hb.prob_in_off))
    out_ep = np.repeat(np.arange(len(ep_names)), np.diff(hb.ep_out_off))
    owner = [names[in_prob[c]] if c < n_in else ep_names[out_ep[c - n_in]] for c in cul]
    print("  culprits of the slow requests:")
    for name, cnt in sorted(zip(*np.unique(owner, return_counts=True)), key=lambda t: -t[1]) if owner else []:
        print(f"    {name:40s} {int(cnt):8d}")
    ex = solver.assemble(hb, np.array(out["assign"]), in_caller, truth=truth_all)["exact"][req]
    edges = np.quantile(cp["latency_us"], np.linspace(0, 1, 11))
    dec = np.clip(np.searchsorted(edges, cp["latency_us"], side="right") - 1, 0, 9)
    print("  exact requests per latency decile: " + " ".join(
        f"{100 * (ex[dec == q] == 1).mean():.1f}%" if (dec == q).any() else "-" for q in range(10)))
cf = None
if args.confidence:
    from traceweaver_b200 import traces
    in_caller = traces.caller_links(ok, hb)
    truth_all = np.concatenate([s.truth.reshape(-1) for s in ok]).astype(np.int32)
    t4 = time.perf_counter()
    cf = solver.request_confidence(hb, out, in_caller)
    t5 = time.perf_counter()
    print(f"request confidence ({1e3 * (t5 - t4):.2f} ms): {cf['requests']} requests")
    print(f"  {'service':28s} {'accuracy':>9s} {'est_accuracy':>13s} {'not_best/n_in':>14s}")
    for p, s in enumerate(ok):
        a = out["assign"][int(hb.prob_tuple_off[p]):int(hb.prob_tuple_off[p + 1])]
        print(f"  {s.name:28s} {100 * accuracy(s, a):8.3f}% {100 * cf['est_accuracy'][p]:12.3f}% "
              f"{100 * out['counters'][p, 0] / s.problem.n_in:13.3f}%")
    req = cf["request"]
    ex = solver.assemble(hb, np.array(out["assign"]), in_caller, truth=truth_all)["exact"][req] == 1
    conf = cf["conf"][req]
    print(f"  expected_exact {cf['expected_exact']:.1f} of {len(req)} requests ({100 * cf['expected_exact'] / max(len(req), 1):.3f} %)"
          f"  exact {int(ex.sum())} ({100 * ex.mean() if len(req) else 0.0:.3f} %)")
    edges = (0.0, 0.5, 0.8, 0.95, 0.99, 1.0)
    print(f"  {'conf bin':16s} {'requests':>9s} {'exact':>8s} {'mean conf':>10s}")
    for lo, hi in zip(edges[:-1], edges[1:]):
        sel = (conf >= lo) & ((conf < hi) if hi < 1.0 else (conf <= hi))
        if sel.any():
            print(f"  [{lo:.2f}, {hi:.2f}{')' if hi < 1.0 else ']'}     {int(sel.sum()):9d} {100 * ex[sel].mean():7.2f}% "
                  f"{100 * conf[sel].mean():9.2f}%")
    if cp is not None:
        n_in = int(hb.prob_in_off[-1])
        names = [s.name for s in ok]
        ep_names = [f"{s.name} -> callee {e}" for s in ok for e in range(s.problem.E)]
        in_prob = np.repeat(np.arange(len(ok)), np.diff(hb.prob_in_off))
        out_ep = np.repeat(np.arange(len(ep_names)), np.diff(hb.ep_out_off))
        slow_req = cp["request"][cp["latency_us"] >= cp["slow_us"]]
        for label, sel in (("confident (conf >= 0.99)", cf["conf"][slow_req] >= 0.99),
                           ("unconfident (conf < 0.99)", cf["conf"][slow_req] < 0.99)):
            cul = cp["culprit"][slow_req[sel]]
            owner = [names[in_prob[c]] if c < n_in else ep_names[out_ep[c - n_in]] for c in cul]
            print(f"  culprits of the slow requests, {label}: {int(sel.sum())}")
            for name, cnt in sorted(zip(*np.unique(owner, return_counts=True)), key=lambda t: -t[1]) if owner else []:
                print(f"    {name:40s} {int(cnt):8d}")
if args.traces:
    from traceweaver_b200 import traces
    in_caller = traces.caller_links(ok, hb)
    truth_all = np.concatenate([s.truth.reshape(-1) for s in ok]).astype(np.int32)
    t4 = time.perf_counter()
    tr = solver.assemble(hb, np.array(out["assign"]), in_caller, truth=truth_all)
    t5 = time.perf_counter()
    ids = [i for s in ok for i in s.in_ids] + [i for s in ok for ids in s.out_ids for i in ids]
    np.savez(args.traces, parent=tr["parent"], root=tr["root"], size=tr["size"], exact=tr["exact"],
             node_trace_id=np.array([t for t, _ in ids]), node_span_id=np.array([sid for _, sid in ids]),
             **({k: cp[k] for k in ("on_path", "self_us", "culprit")} if cp is not None else {}),
             **({k: cf[k] for k in ("conf", "weakest", "p")} if cf is not None else {}))
    n_in = int(hb.prob_in_off[-1])
    requests = int((tr["exact"] >= 0).sum())
    e2e = end_to_end_accuracy([[t for t, _ in s.in_ids] for s in ok], [s.truth for s in ok],
                              [out["assign"][int(hb.prob_tuple_off[p]):int(hb.prob_tuple_off[p + 1])]
                               for p in range(len(ok))])
    print(f"request trees ({1e3 * (t5 - t4):.2f} ms, with the truth join): {requests} requests, "
          f"{int((tr['size'][n_in:] > 0).sum())} detached fragments, {int((tr['root'] < 0).sum())} nodes on cycles; "
          f"exact {100 * (tr['exact'] == 1).sum() / max(requests, 1):7.3f} %  end-to-end accuracy {100 * e2e:7.3f} %"
          f"  -> {args.traces}")
