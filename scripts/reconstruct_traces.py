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
node_span_id; it prints the share of exact requests beside the end-to-end accuracy."""
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
out = solver.solve(hb, want_likelihood=args.likelihood, want_mixtures=args.likelihood)
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
if args.traces:
    from traceweaver_b200 import traces
    in_caller = traces.caller_links(ok, hb)
    truth_all = np.concatenate([s.truth.reshape(-1) for s in ok]).astype(np.int32)
    t4 = time.perf_counter()
    tr = solver.assemble(hb, np.array(out["assign"]), in_caller, truth=truth_all)
    t5 = time.perf_counter()
    ids = [i for s in ok for i in s.in_ids] + [i for s in ok for ids in s.out_ids for i in ids]
    np.savez(args.traces, parent=tr["parent"], root=tr["root"], size=tr["size"], exact=tr["exact"],
             node_trace_id=np.array([t for t, _ in ids]), node_span_id=np.array([sid for _, sid in ids]))
    n_in = int(hb.prob_in_off[-1])
    requests = int((tr["exact"] >= 0).sum())
    e2e = end_to_end_accuracy([[t for t, _ in s.in_ids] for s in ok], [s.truth for s in ok],
                              [out["assign"][int(hb.prob_tuple_off[p]):int(hb.prob_tuple_off[p + 1])]
                               for p in range(len(ok))])
    print(f"request trees ({1e3 * (t5 - t4):.2f} ms, with the truth join): {requests} requests, "
          f"{int((tr['size'][n_in:] > 0).sum())} detached fragments, {int((tr['root'] < 0).sum())} nodes on cycles; "
          f"exact {100 * (tr['exact'] == 1).sum() / max(requests, 1):7.3f} %  end-to-end accuracy {100 * e2e:7.3f} %"
          f"  -> {args.traces}")
