"""Time-compressed services through the float64 path (tw_engine_bind_f64), one JSON line.

    python scripts/time_float_times.py [--services 2016] [--n-in 1250] [--seed 0] [--sample 108]

executor.py --compress_factor as exps/exp5 runs it: the alibaba-shaped blocks generated uncompressed (one
request per second) and each service's start times divided by its factor in float64, durations kept, so
the engine sees fractional microseconds.  The factor is the load bench.py's integer alibaba stream generates
at (shard.stream_spec).  Reports spans/s through BatchSolver (wall clock incl. staging, H2D and D2H), the
device time of the two conversion kernels (torch.profiler, in a run of its own) and engine == the float64
build of the oracle (tests/oracle_f64.py) on a sample, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def compressed_blocks(n_services, n_in, seed):
    from traceweaver_b200 import shard, synth
    from traceweaver_b200.batch import ServiceBlock
    blocks = []
    for b in shard.stream_spec("alibaba", n_services, n_in, seed):
        blk = synth.make_block(b.shape, b.services, b.n_in, 1.0, b.seed, quantum_us=b.quantum_us)
        f = lambda a, cf=float(b.load): a.astype(np.float64) / cf
        blocks.append(ServiceBlock(in_start=f(blk.in_start), in_end=f(blk.in_start) + (blk.in_end - blk.in_start),
                                   out_start=[f(o) for o in blk.out_start],
                                   out_end=[f(o) + (e - o) for o, e in zip(blk.out_start, blk.out_end)],
                                   preds=blk.preds, truth=blk.truth, name=blk.name))
    return blocks


def first_services(blocks, per):
    from traceweaver_b200.batch import ServiceBlock
    return [ServiceBlock(in_start=b.in_start[:per], in_end=b.in_end[:per], out_start=[o[:per] for o in b.out_start],
                         out_end=[o[:per] for o in b.out_end], preds=b.preds, truth=b.truth[:, :per], name=b.name)
            for b in blocks]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--services", type=int, default=2016)
    ap.add_argument("--n-in", type=int, default=1250)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--sample", type=int, default=108)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import oracle_f64
    from traceweaver_b200 import synth
    from traceweaver_b200.api import BatchSolver
    from traceweaver_b200.batch import build_batch_from_blocks
    from traceweaver_b200.engine import Engine
    from traceweaver_b200.predictor import solve_bound

    blocks = compressed_blocks(args.services, args.n_in, args.seed)
    hb = build_batch_from_blocks(blocks)
    n_spans = synth.span_count(blocks)
    solver = BatchSolver(device=0, seed_select=10)
    solver.solve(hb)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.reps):
        out = solver.solve(hb)
    ms = (time.perf_counter() - t0) * 1e3 / args.reps
    solver.close()
    acc = float((out["assign"] == synth.truth_assign(blocks)).mean())

    # the conversion kernels alone: re-bind the resident batch under the profiler
    eng = Engine(0)
    eng.bind(hb)
    d = eng.d
    torch.cuda.synchronize()
    binds = 5
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(binds):
            eng.bind(hb, device_arrays=d)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        for name in ("k_time_shift", "k_to_fixed"):
            if name in ev.key:
                t = getattr(ev, "device_time_total", None)
                kern[name] = kern.get(name, 0.0) + (t if t is not None else ev.cuda_time_total) / binds / 1e3

    # engine == float64 oracle on the first services of every block
    per = max(1, args.sample // len(blocks))
    shb = build_batch_from_blocks(first_services(blocks, per))
    eng.bind(shb)
    res = solve_bound(eng)
    ref = oracle_f64.find_assignments(shb, 10, threads=os.cpu_count() or 1)
    ob = oracle_f64.OracleBatch(shb)
    g0 = ob.params_pass0()
    ref0 = ob.stitch(ob.score(gauss=g0)["cut"], gauss=g0, want_topk=False)["assign"]
    same = bool(np.array_equal(res["assign"].cpu().numpy(), ref["assign"]))
    same0 = bool(np.array_equal(res["assign_pass0"].cpu().numpy(), ref0))
    eng.close()
    spans_read = int(hb.prob_in_off[-1]) + int(hb.ep_out_off[-1])
    print(json.dumps({
        "workload": "alibaba-shaped services with float64 start times divided by their compression factor "
                    "(executor.py --compress_factor, exps/exp5), one call through BatchSolver",
        "card": card(), "services": hb.n_problems, "spans": n_spans, "ms_per_call": round(ms, 3),
        "e2e_spans_per_s": n_spans / (ms * 1e-3), "accuracy": acc,
        "conversion_kernels_ms": {k: round(v, 4) for k, v in kern.items()},
        "conversion_read_bytes_per_kernel": 16 * spans_read,
        "engine_equals_float_oracle_on_sample": same,
        "engine_equals_float_oracle_iteration0_on_sample": same0,
        "sample": f"first {per} services of each of the {len(blocks)} blocks ({shb.n_problems} services)"}))


if __name__ == "__main__":
    main()
