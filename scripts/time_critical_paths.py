"""Time tw_critical_paths (the join, the level walk, the culprits and the per-service sums) on a generated
two-tier hotel deployment.

    python scripts/time_critical_paths.py [--replicas 4096] [--requests 1000] [--reps 20] [--out result.json]

synth.hotel_tree (seeded): `replicas` x `requests` requests of 7 nodes each (frontend and search in-spans,
five out-spans).  The whole call, traces.critical_paths with the span arrays already on the device, is timed
with CUDA events over --reps calls after a warm-up, on the true assignment and on a BatchSolver.solve result;
each call reads back the join's error words (one small copy and a stream synchronise).  The split between
kernels comes from a separate torch.profiler run.  The card's name and power limit are read in the same run.

Algorithmic bytes of one call (N nodes, n_in in-spans, n_tuple = sum n_in * E, R join rounds that ran,
Lr walk levels that ran after level 0, V on-path in-spans, W on-path out-spans, C their callee in-spans on
the path, K children the walked in-spans have):
  join     as scripts/time_traces.py: 4 n_tuple + 4 claimed + 8 n_in + 4 linked + 8 n_out + 4 N + 12 N R + 16 N
  memsets  9 N (on_path, self_us) + 12 n_in (level words, culprit maxima)
  walk     8 n_in (level 0: root read, culprit written) + 4 n_in Lr (level words scanned) + per walked in-span
           16 (window or times) + 4 E (assign) + 9 (self, on_path) + 16 per child (times) + per on-path
           out-span 4 (claim) + 9 + per on-path callee 16 (times) + 20 (window, level)
  culprit  2 N (on_path twice) + 2 x 20 per on-path node (root, self, maximum)
  sums     N (on_path) + 13 per on-path node (self, root, slow flag)
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
    sys.exit("time_critical_paths.py measures on the GPU; there is no CPU measurement")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.max.mem",
                       "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
tree = synth.hotel_tree(args.replicas, args.requests, args.load, seed=args.seed)
hb = tree["hb"]
n_in, n_out = int(hb.prob_in_off[-1]), int(hb.ep_out_off[-1])
N, n_tuple = n_in + n_out, int(hb.prob_tuple_off[-1])
E_of_in = np.repeat(np.diff(hb.prob_ep_off), np.diff(hb.prob_in_off))

solver = BatchSolver(device=0)
solved = np.array(solver.solve(hb)["assign"])
eng = solver.engine
eng.lib.tw_debug_trace_rounds.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
eng.lib.tw_debug_critical_levels.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
d = _to_device(dict(truth=tree["truth"], solved=solved, in_caller=tree["in_caller"]), eng.device)
spans = traces.upload_spans(eng, hb)
slow_us = traces.lower_quantile(traces.request_latencies(spans, d["in_caller"])[1], 0.99)


def debug():
    launched, run, levels = C.c_int(0), C.c_int(0), C.c_int(0)
    eng.lib.tw_debug_trace_rounds(eng.h, C.byref(launched), C.byref(run))
    eng.lib.tw_debug_critical_levels(eng.h, C.byref(levels))
    return launched.value, run.value, levels.value


def algo_bytes(assign, res, run):
    claimed = int((assign >= 0).sum())
    linked = int((tree["in_caller"] >= 0).sum())
    join = 4 * n_tuple + 4 * claimed + 8 * n_in + 4 * linked + 8 * n_out + 4 * N + 12 * N * run + 16 * N
    on = res["on_path"].cpu().numpy() == 1
    V, W = int(on[:n_in].sum()), int(on[n_in:].sum())
    walked_E = int(E_of_in[on[:n_in]].sum())
    kids = int((assign.reshape(-1) >= 0).sum())              # an upper bound: the walked in-spans' children
    C_on = V - int(res["requests"][0].item())
    depth_levels = 1                                          # levels after level 0 that ran (hotel: search)
    walk = 8 * n_in + 4 * n_in * depth_levels + V * (16 + 9) + 4 * walked_E + 16 * kids + W * (4 + 9) + C_on * 36
    return join + 9 * N + 12 * n_in + walk + 2 * N + 40 * (V + W) + N + 13 * (V + W)


def timed(name):
    fn = lambda: traces.critical_paths(eng, hb, d[name], d["in_caller"], slow_us, spans=spans)
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
    launched, run, levels = debug()
    c0 = eng.launch_count()
    fn()
    launches = eng.launch_count() - c0
    eng.status()
    nbytes = algo_bytes(d[name].cpu().numpy(), res, run)
    on = res["on_path"].cpu().numpy()
    return dict(ms=round(ms, 4), rounds_launched=launched, rounds_run=run, levels=levels, launches=launches,
                requests=int(res["requests"][0]), slow_requests=int(res["requests"][1]),
                on_path_nodes=int(on.sum()), algo_bytes=nbytes, gbps=round(nbytes / ms / 1e6, 1),
                hbm_share=round(nbytes / (ms * 1e-3) / HBM_PEAK, 4))


res = dict(truth=timed("truth"), solved=timed("solved"))

from torch.profiler import ProfilerActivity, profile
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(5):
        traces.critical_paths(eng, hb, d["solved"], d["in_caller"], slow_us, spans=spans)
    torch.cuda.synchronize()
kern = {}
for ev in prof.key_averages():
    for k in ("k_link_out", "k_link_in", "k_jump", "k_roots", "k_cp_level", "k_cp_culprit_max",
              "k_cp_culprit_min", "k_cp_reduce", "Memset"):
        if k in ev.key:
            kern[k] = round(kern.get(k, 0.0) + ev.device_time_total / 1e3 / 5, 4)
solver.close()

out = dict(card=card, requests=args.replicas * args.requests, in_spans=n_in, out_spans=n_out, nodes=N,
           slow_us=slow_us, kernel_ms_per_call=kern, **res)
print(json.dumps(out, indent=1))
if args.out:
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
