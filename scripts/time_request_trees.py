"""Time the request-tree entry points on a generated two-tier hotel deployment: tw_assemble_traces (the join
by pointer jumping), tw_critical_paths (the join, the level walk, the culprits and the per-service sums) and
tw_request_confidence (the join, the per-in-span step, the per-request pass and the sums).

    python scripts/time_request_trees.py [--replicas 4096] [--requests 1000] [--reps 20] [--out result.json]

The bench streams are independent services without RPC links, so this script generates its own:
synth.hotel_tree (seeded), `replicas` x `requests` requests, each a frontend call to search (which calls
geo and rate), reservation and profile: 2 in-spans and 5 out-spans, 7 nodes per request.  One
BatchSolver.solve(want_likelihood=True, want_scores=True, want_mixtures=True) gives the solved assignment, its
chosen tuples' scores and the final top-K; the true assignment is scored with BatchSolver.score under the
same mixtures.  Each call (traces.assemble, traces.critical_paths, traces.request_confidence) is timed whole,
with every input already on the device, with CUDA events over --reps calls after a warm-up, on the true and
on the solved assignment.  Each call reads back the join's error words (one small copy and a stream
synchronise; request_confidence also its size check).  The split between kernels comes from a separate
torch.profiler run per call.  The card's name and power limit are read in the same run.

Algorithmic bytes of one call (N = n_in + n_out nodes, n_tuple = sum n_in * E, R join rounds that ran):
  join     4 n_tuple (assign) + 4 claimed out-spans (parent) + 8 n_in (in_caller, parent) + 4 linked in-spans
           (claim word); the memsets 8 n_out + 4 N; 12 N per round that runs (the node's ancestor and the
           ancestor's ancestor read, the new one written); roots 16 N (ancestor, its parent, root written,
           size incremented).  All three calls run it.
critical_paths, besides the join (Lr walk levels that ran after level 0, V on-path in-spans, W on-path
out-spans, C their callee in-spans on the path, K children the walked in-spans have):
  memsets  9 N (on_path, self_us) + 12 n_in (level words, culprit maxima)
  walk     8 n_in (level 0: root read, culprit written) + 4 n_in Lr (level words scanned) + per walked in-span
           16 (window or times) + 4 E (assign) + 9 (self, on_path) + 16 per child (times) + per on-path
           out-span 4 (claim) + 9 + per on-path callee 16 (times) + 20 (window, level)
  culprit  2 N (on_path twice) + 2 x 20 per on-path node (root, self, maximum)
  sums     N (on_path) + 13 per on-path node (self, root, slow flag)
request_confidence, besides the join (E callees of an in-span's service, Q request roots):
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
from torch.profiler import ProfilerActivity, profile
from traceweaver_b200 import synth, traces
from traceweaver_b200.api import BatchSolver
from traceweaver_b200.engine import _to_device

if not torch.cuda.is_available():
    sys.exit("time_request_trees.py measures on the GPU; there is no CPU measurement")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.max.mem",
                       "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
tree = synth.hotel_tree(args.replicas, args.requests, args.load, seed=args.seed)
hb = tree["hb"]
n_in, n_out = int(hb.prob_in_off[-1]), int(hb.ep_out_off[-1])
N, n_tuple = n_in + n_out, int(hb.prob_tuple_off[-1])
E_of_in = np.repeat(np.diff(hb.prob_ep_off), np.diff(hb.prob_in_off))

solver = BatchSolver(device=0)
out = {k: np.array(v) for k, v in solver.solve(hb, want_likelihood=True, want_scores=True,
                                                 want_mixtures=True).items()}
sc = solver.score(hb, tree["truth"], out["mixtures"])
eng = solver.engine
eng.lib.tw_debug_trace_rounds.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
eng.lib.tw_debug_critical_levels.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
d = _to_device(dict(truth=tree["truth"], solved=out["assign"], in_caller=tree["in_caller"],
                    solved_score=out["chosen_score"], solved_code=out["chosen_code"], truth_score=sc["score"],
                    truth_code=sc["code"], topk_score=out["topk_score"], topk_idx=out["topk_idx"],
                    topk_cnt=out["topk_cnt"]), eng.device)
topk = {k: d[k] for k in ("topk_score", "topk_idx", "topk_cnt")}
spans = traces.upload_spans(eng, hb)
slow_us = traces.lower_quantile(traces.request_latencies(spans, d["in_caller"])[1], 0.99)

CALLS = {
    "assemble": lambda name: traces.assemble(eng, hb, d[name], d["in_caller"]),
    "critical_paths": lambda name: traces.critical_paths(eng, hb, d[name], d["in_caller"], slow_us, spans=spans),
    "request_confidence": lambda name: traces.request_confidence(eng, hb, d[name], d["in_caller"],
                                                                 d[name + "_score"], d[name + "_code"], topk),
}
JOIN_KERNELS = ("k_link_out", "k_link_in", "k_jump", "k_roots")
KERNELS = {"assemble": JOIN_KERNELS,
           "critical_paths": JOIN_KERNELS + ("k_cp_level", "k_cp_culprit_max", "k_cp_culprit_min", "k_cp_reduce",
                                             "Memset"),
           "request_confidence": JOIN_KERNELS + ("k_conf_step", "k_conf_root", "k_conf_reduce", "k_conf_total",
                                                 "Memset")}


def join_bytes(assign, run):
    claimed = int((assign >= 0).sum())
    linked = int((tree["in_caller"] >= 0).sum())
    return 4 * n_tuple + 4 * claimed + 8 * n_in + 4 * linked + 8 * n_out + 4 * N + 12 * N * run + 16 * N


def paths_bytes(assign, res, run):
    on = res["on_path"].cpu().numpy() == 1
    V, W = int(on[:n_in].sum()), int(on[n_in:].sum())
    walked_E = int(E_of_in[on[:n_in]].sum())
    kids = int((assign.reshape(-1) >= 0).sum())              # an upper bound: the walked in-spans' children
    C_on = V - int(res["requests"][0].item())
    depth_levels = 1                                          # levels after level 0 that ran (hotel: search)
    walk = 8 * n_in + 4 * n_in * depth_levels + V * (16 + 9) + 4 * walked_E + 16 * kids + W * (4 + 9) + C_on * 36
    return join_bytes(assign, run) + 9 * N + 12 * n_in + walk + 2 * N + 40 * (V + W) + N + 13 * (V + W)


def confidence_bytes(assign, run, roots):
    step = 24 * n_tuple + (50 + 4 + 20 + 20) * n_in
    request = 36 * n_in + 20 * roots
    sums = 12 * n_in + 8 * roots
    return join_bytes(assign, run) + 24 * n_in + step + request + sums


def timed(call, name):
    fn = lambda: CALLS[call](name)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.reps):
        fn()
    b.record()
    b.synchronize()
    ms = a.elapsed_time(b) / args.reps
    launched, run, levels = C.c_int(0), C.c_int(0), C.c_int(0)
    eng.lib.tw_debug_trace_rounds(eng.h, C.byref(launched), C.byref(run))
    eng.lib.tw_debug_critical_levels(eng.h, C.byref(levels))
    c0 = eng.launch_count()
    res = fn()
    launches = eng.launch_count() - c0
    eng.status()
    assign = d[name].cpu().numpy()
    row = dict(ms=round(ms, 4), rounds_launched=launched.value, rounds_run=run.value)
    if call == "assemble":
        size, root = res["size"].cpu().numpy(), res["root"].cpu().numpy()
        nbytes = join_bytes(assign, run.value)
        row.update(launches=launches, in_span_roots=int((size[:n_in] > 0).sum()),
                   detached_roots=int((size[n_in:] > 0).sum()), on_cycles=int((root < 0).sum()))
    elif call == "critical_paths":
        nbytes = paths_bytes(assign, res, run.value)
        row.update(levels=levels.value, launches=launches, requests=int(res["requests"][0]),
                   slow_requests=int(res["requests"][1]), on_path_nodes=int(res["on_path"].cpu().numpy().sum()))
    else:
        roots = int(res["requests"][0])
        nbytes = confidence_bytes(assign, run.value, roots)
        row.update(launches=launches, requests=roots, expected_exact=float(res["expected_exact"][0]))
    row.update(algo_bytes=nbytes, gbps=round(nbytes / ms / 1e6, 1), hbm_share=round(nbytes / (ms * 1e-3) / HBM_PEAK, 4))
    return row


def kernel_ms(call):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            CALLS[call]("solved")
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        for k in KERNELS[call]:
            if k in ev.key:
                kern[k] = round(kern.get(k, 0.0) + ev.device_time_total / 1e3 / 5, 4)
    return kern


res = {call: dict(truth=timed(call, "truth"), solved=timed(call, "solved")) for call in CALLS}
for call in CALLS:
    res[call]["kernel_ms_per_call"] = kernel_ms(call)
solver.close()

result = dict(card=card, requests=args.replicas * args.requests, in_spans=n_in, out_spans=n_out, nodes=N,
              services=hb.n_problems, slow_us=slow_us, **res)
print(json.dumps(result, indent=1))
if args.out:
    with open(args.out, "w") as f:
        json.dump(result, f, indent=1)
