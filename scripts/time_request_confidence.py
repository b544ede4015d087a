"""Time tw_request_confidence (the join, the per-in-span step, the per-request pass and the sums) on a
generated two-tier hotel deployment.

    python scripts/time_request_confidence.py [--replicas 4096] [--requests 1000] [--reps 20] [--out result.json]

synth.hotel_tree (seeded): `replicas` x `requests` requests of 7 nodes each (frontend and search in-spans,
five out-spans).  One BatchSolver.solve(want_likelihood=True, want_scores=True) gives the chosen tuples'
scores and the final top-K.  The whole call, traces.request_confidence with every input already on the
device, is timed with CUDA events over --reps calls after a warm-up, on that solve result and on the truth
(scored with BatchSolver.score); each call reads back the join's error words and the size check (two small
copies, each with a stream synchronise).  The split between kernels comes from a separate torch.profiler run.
The card's name and power limit are read in the same run.

Algorithmic bytes of one call (N nodes, n_in in-spans, E callees of an in-span's service, n_tuple = sum n_in E,
R join rounds that ran, Q request roots):
  join     as scripts/time_traces.py: 4 n_tuple + 4 claimed + 8 n_in + 4 linked + 8 n_out + 4 N + 12 N R + 16 N
  memsets  24 n_in (decisions, zero, log_conf, smallest p bits)
  step     per in-span 24 E (assign, top-K tuples) + 50 (score, code, top-K scores and count) + 4 (root)
           + 20 (p, ell, weakest written) + 20 (its root's decision, sum and p-bits atomics)
  request  per in-span 20 (root, p, the root's p bits) + 16 (conf, weakest_p written); per root 20 (zero,
           log_conf, decisions, weakest)
  sums     per in-span 12 (p, root) + per root 8 (conf)
quoted against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s)."""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import numpy as np

HBM_PEAK = 3.35e12

ap = argparse.ArgumentParser()
ap.add_argument("--replicas", type=int, default=4096)
ap.add_argument("--requests", type=int, default=1000)
ap.add_argument("--load", type=float, default=100.0)
ap.add_argument("--seed", type=int, default=10)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--out", default=None)
args = ap.parse_args()

import torch
from traceweaver_b200 import synth, traces
from traceweaver_b200.api import BatchSolver
from traceweaver_b200.engine import _to_device

if not torch.cuda.is_available():
    sys.exit("time_request_confidence.py measures on the GPU; there is no CPU measurement")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.max.mem",
                       "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
tree = synth.hotel_tree(args.replicas, args.requests, args.load, seed=args.seed)
hb = tree["hb"]
n_in, n_out = int(hb.prob_in_off[-1]), int(hb.ep_out_off[-1])
N, n_tuple = n_in + n_out, int(hb.prob_tuple_off[-1])

solver = BatchSolver(device=0)
out = {k: np.array(v) for k, v in solver.solve(hb, want_likelihood=True, want_scores=True,
                                                 want_mixtures=True).items()}
sc = solver.score(hb, tree["truth"], out["mixtures"])
eng = solver.engine
eng.lib.tw_debug_trace_rounds.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
d = _to_device(dict(truth=tree["truth"], solved=out["assign"], in_caller=tree["in_caller"],
                    solved_score=out["chosen_score"], solved_code=out["chosen_code"], truth_score=sc["score"],
                    truth_code=sc["code"], topk_score=out["topk_score"], topk_idx=out["topk_idx"],
                    topk_cnt=out["topk_cnt"]), eng.device)
topk = {k: d[k] for k in ("topk_score", "topk_idx", "topk_cnt")}


def algo_bytes(assign, run, roots):
    claimed = int((assign >= 0).sum())
    linked = int((tree["in_caller"] >= 0).sum())
    join = 4 * n_tuple + 4 * claimed + 8 * n_in + 4 * linked + 8 * n_out + 4 * N + 12 * N * run + 16 * N
    step = 24 * n_tuple + (50 + 4 + 20 + 20) * n_in
    request = 36 * n_in + 20 * roots
    sums = 12 * n_in + 8 * roots
    return join + 24 * n_in + step + request + sums


def timed(name):
    fn = lambda: traces.request_confidence(eng, hb, d[name], d["in_caller"], d[name + "_score"], d[name + "_code"],
                                           topk)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.reps):
        res = fn()
    b.record()
    b.synchronize()
    ms = a.elapsed_time(b) / args.reps
    launched, run = C.c_int(0), C.c_int(0)
    eng.lib.tw_debug_trace_rounds(eng.h, C.byref(launched), C.byref(run))
    c0 = eng.launch_count()
    fn()
    launches = eng.launch_count() - c0
    roots = int(res["requests"][0])
    nbytes = algo_bytes(d[name].cpu().numpy(), run.value, roots)
    return dict(ms=round(ms, 4), rounds_launched=launched.value, rounds_run=run.value, launches=launches,
                requests=roots, expected_exact=float(res["expected_exact"][0]), algo_bytes=nbytes,
                gbps=round(nbytes / ms / 1e6, 1), hbm_share=round(nbytes / (ms * 1e-3) / HBM_PEAK, 4))


res = dict(solved=timed("solved"), truth=timed("truth"))

from torch.profiler import ProfilerActivity, profile
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(5):
        traces.request_confidence(eng, hb, d["solved"], d["in_caller"], d["solved_score"], d["solved_code"], topk)
    torch.cuda.synchronize()
kern = {}
for ev in prof.key_averages():
    for k in ("k_link_out", "k_link_in", "k_jump", "k_roots", "k_conf_step", "k_conf_root", "k_conf_reduce",
              "k_conf_total", "Memset"):
        if k in ev.key:
            kern[k] = round(kern.get(k, 0.0) + ev.device_time_total / 1e3 / 5, 4)
solver.close()

result = dict(card=card, requests=args.replicas * args.requests, in_spans=n_in, out_spans=n_out, nodes=N,
              services=hb.n_problems, kernel_ms_per_call=kern, **res)
print(json.dumps(result, indent=1))
if args.out:
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
