"""Time tw_score_assignments (k_assess + k_assess_reduce) on the bench workload and the extra time
want_likelihood=True adds to a BatchSolver.solve call.

    python scripts/time_score_assign.py [--services 8192] [--n-in 1000] [--reps 50] [--out result.json]

Kernel time: CUDA events around Engine.score_assignments (the two kernels, nothing else on an int64 bind),
averaged over --reps calls after a warm-up; the split between the two kernels comes from a separate
torch.profiler run.  Bytes are the algorithm's gathers and writes per in-span with E callees: the tuple's
indices (4E), the in-span (16), the chosen spans (16E), the final top-K row for the margin (5 * (8 + 4E)
and its count) and the outputs (17); quoted against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s)."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

HBM_PEAK = 3.35e12

ap = argparse.ArgumentParser()
ap.add_argument("--services", type=int, default=8192)
ap.add_argument("--n-in", type=int, default=1000)
ap.add_argument("--reps", type=int, default=50)
ap.add_argument("--solve-rounds", type=int, default=6)
ap.add_argument("--out", default=None)
args = ap.parse_args()

import torch
from traceweaver_b200 import synth
from traceweaver_b200.api import BatchSolver
from traceweaver_b200.batch import build_batch_from_blocks
from traceweaver_b200.engine import Engine
from traceweaver_b200.predictor import solve_bound

if not torch.cuda.is_available():
    sys.exit("time_score_assign.py measures on the GPU; there is no CPU measurement")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,clocks.max.mem",
                       "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
hb = build_batch_from_blocks(synth.hotel_stream(args.services, args.n_in))
n_in = int(hb.prob_in_off[-1])
E = np.repeat(np.diff(hb.prob_ep_off), np.diff(hb.prob_in_off)).astype(np.int64)
bytes_no_margin = int(np.sum(4 * E + 16 + 16 * E + 17 - 8))      # no margin: 9 B written
bytes_margin = int(np.sum(4 * E + 16 + 16 * E + 5 * (8 + 4 * E) + 1 + 17))

eng = Engine(0)
eng.bind(hb)
res = solve_bound(eng)
p1, assign = res["params_pass1"], res["assign"]
top = dict(topk_score=res["topk_score"], topk_idx=res["topk_idx"], topk_cnt=res["topk_cnt"])


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


ms_margin = timed(lambda: eng.score_assignments(p1, assign, final_topk=top), args.reps)
ms_plain = timed(lambda: eng.score_assignments(p1, assign), args.reps)
c0 = eng.launch_count()
eng.score_assignments(p1, assign, final_topk=top)
launches = eng.launch_count() - c0
eng.status()

# per-kernel split, in a run of its own
from torch.profiler import ProfilerActivity, profile
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(10):
        eng.score_assignments(p1, assign, final_topk=top)
    torch.cuda.synchronize()
kern = {}
for ev in prof.key_averages():
    if "k_assess" in ev.key:
        kern["k_assess_reduce" if "reduce" in ev.key else "k_assess"] = ev.device_time_total / 1e3 / 10
eng.close()

# what want_likelihood adds to a whole solve: alternate the two calls
solver = BatchSolver(device=0)
solver.solve(hb)
solver.solve(hb, want_likelihood=True)
t_off, t_on = [], []
for _ in range(args.solve_rounds):
    for want, acc in ((False, t_off), (True, t_on)):
        torch.cuda.synchronize()
        t = time.perf_counter()
        solver.solve(hb, want_likelihood=want)
        acc.append(1e3 * (time.perf_counter() - t))
solver.close()

out = dict(card=card, services=hb.n_problems, in_spans=n_in, launches_per_call=launches,
           ms_with_margin=round(ms_margin, 4), ms_without_margin=round(ms_plain, 4),
           kernel_ms=({k: round(v, 4) for k, v in kern.items()}),
           bytes_with_margin=bytes_margin, bytes_without_margin=bytes_no_margin,
           gbps_with_margin=round(bytes_margin / ms_margin / 1e6, 1),
           gbps_without_margin=round(bytes_no_margin / ms_plain / 1e6, 1),
           hbm_share_with_margin=round(bytes_margin / (ms_margin * 1e-3) / HBM_PEAK, 4),
           hbm_share_without_margin=round(bytes_no_margin / (ms_plain * 1e-3) / HBM_PEAK, 4),
           solve_ms_off=[round(x, 2) for x in t_off], solve_ms_on=[round(x, 2) for x in t_on],
           solve_ms_off_median=round(float(np.median(t_off)), 2), solve_ms_on_median=round(float(np.median(t_on)), 2))
print(json.dumps(out, indent=1))
if args.out:
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
