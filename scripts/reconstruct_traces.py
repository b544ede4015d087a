"""Reconstruct a directory of Jaeger JSON traces end to end: loader -> batch engine -> accuracy.

    python scripts/reconstruct_traces.py <trace dir> [--layout hotel|media|node|alibaba] [--device 0] [--likelihood]

Prints, per solved service, the assignment accuracy against the traces' own parent links
(the reference's AccuracyForService, helpers/utils.py:34-60) and the time of each stage — the same
numbers executor.py prints for `--predictor_indices 10`.  --likelihood adds, per service, the mean
log-likelihood of the chosen tuples under the refitted delay model, quantiles of the margin to the runner-up
(or to the best tuple, for an in-span that did not get its best), and for the wrong in-spans whether the
true tuple scores above the chosen one (a search error: the window's MWIS and deletion pushed it out),
below it (a model error), or is infeasible."""
import argparse, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("directory")
ap.add_argument("--layout", default="hotel", choices=["hotel", "media", "node", "alibaba"])
ap.add_argument("--device", type=int, default=0)
ap.add_argument("--seed", type=int, default=10)
ap.add_argument("--likelihood", action="store_true", help="print per-service confidence and error classes")
args = ap.parse_args()

from traceweaver_b200.api import BatchSolver
from traceweaver_b200.loader import load_jaeger_dir, to_host_batch, accuracy

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
