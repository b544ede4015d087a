"""Time tw_assemble_traces (request trees by pointer jumping) on a generated two-tier hotel deployment.

    python scripts/time_traces.py [--replicas 4096] [--requests 1000] [--reps 20] [--out result.json]

The bench streams are independent services without RPC links, so this script generates its own:
synth.hotel_tree (seeded), `replicas` x `requests` requests, each a frontend call to search (which calls
geo and rate), reservation and profile: 2 in-spans and 5 out-spans, 7 nodes per request.  The join is
timed with CUDA events around traces.assemble over --reps calls after a warm-up, on the true assignment
and on a BatchSolver.solve result; each call ends by reading back its error words (one small copy and a
stream synchronise).  The split between kernels comes from a separate torch.profiler run.

Algorithmic bytes of one call (n_tuple = sum n_in * E, N = n_in + n_out nodes, R = rounds that ran):
  links    4 n_tuple (assign) + 4 claimed out-spans (parent) + 8 n_in (in_caller, parent) + 4 linked in-spans
           (claim word); the memsets 8 n_out + 4 N
  rounds   12 N per round that runs: the node's ancestor and the ancestor's ancestor read, the new one written
  roots    16 N: ancestor, its parent, root written, size incremented
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
    sys.exit("time_traces.py measures on the GPU; there is no CPU measurement")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.max.mem",
                       "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
tree = synth.hotel_tree(args.replicas, args.requests, args.load, seed=args.seed)
hb = tree["hb"]
n_in, n_out = int(hb.prob_in_off[-1]), int(hb.ep_out_off[-1])
N, n_tuple = n_in + n_out, int(hb.prob_tuple_off[-1])

solver = BatchSolver(device=0)
solved = np.array(solver.solve(hb)["assign"])
eng = solver.engine
eng.lib.tw_debug_trace_rounds.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
d = _to_device(dict(truth=tree["truth"], solved=solved, in_caller=tree["in_caller"]), eng.device)


def rounds():
    launched, run = C.c_int(0), C.c_int(0)
    eng.lib.tw_debug_trace_rounds(eng.h, C.byref(launched), C.byref(run))
    return launched.value, run.value


def algo_bytes(assign, run):
    claimed = int((assign >= 0).sum())
    linked = int((tree["in_caller"] >= 0).sum())
    return 4 * n_tuple + 4 * claimed + 8 * n_in + 4 * linked + 8 * n_out + 4 * N + 12 * N * run + 16 * N


def timed(name, host_assign):
    fn = lambda: traces.assemble(eng, hb, d[name], d["in_caller"])
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
    launched, run = rounds()
    c0 = eng.launch_count()
    fn()
    launches = eng.launch_count() - c0
    nbytes = algo_bytes(host_assign, run)
    size = res["size"].cpu().numpy()
    root = res["root"].cpu().numpy()
    return dict(ms=round(ms, 4), rounds_launched=launched, rounds_run=run, launches=launches,
                in_span_roots=int((size[:n_in] > 0).sum()), detached_roots=int((size[n_in:] > 0).sum()),
                on_cycles=int((root < 0).sum()), algo_bytes=nbytes, gbps=round(nbytes / ms / 1e6, 1),
                hbm_share=round(nbytes / (ms * 1e-3) / HBM_PEAK, 4))


res = dict(truth=timed("truth", tree["truth"]), solved=timed("solved", solved))

from torch.profiler import ProfilerActivity, profile
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(5):
        traces.assemble(eng, hb, d["solved"], d["in_caller"])
    torch.cuda.synchronize()
kern = {}
for ev in prof.key_averages():
    for k in ("k_link_out", "k_link_in", "k_jump", "k_roots"):
        if k in ev.key:
            kern[k] = round(ev.device_time_total / 1e3 / 5, 4)
solver.close()

out = dict(card=card, requests=args.replicas * args.requests, in_spans=n_in, out_spans=n_out, nodes=N,
           kernel_ms_per_call=kern, **res)
print(json.dumps(out, indent=1))
if args.out:
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
