"""What want_likelihood=True adds to the cache-mode leg: the 9 golden cache-mode services (skip budgets > 0)
through skipmode.solve, as bench.py's cache leg runs them, with and without the likelihood, alternated.

    python scripts/time_skip_score_assign.py [--reps 5]

Prints the card, its power limit and one JSON line: the median over reps of the leg's total ms each way."""
import argparse
import glob
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    from golden_util import Golden
    from traceweaver_b200 import skipmode
    from traceweaver_b200.engine import Engine
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    gs = [Golden(f) for f in sorted(glob.glob(os.path.join(ROOT, "tests", "golden_cache", "*__*.npz")))]
    gs = [g for g in gs if any(v != 0 for v in g.meta["skip_budget"].values())]
    eng = Engine(0)

    def leg(want):
        total = 0.0
        for g in gs:
            prob = g.problem()
            st = skipmode.SkipState()
            st.time_windows = [tuple(w) for w in g.meta["time_windows_before"]]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            skipmode.solve(eng, prob.in_start, prob.in_end, prob.out_start, prob.out_end, prob.preds,
                           labels=[g.meta["in_ep"]] + g.topo, state=st, want_topk=False, want_likelihood=want)
            total += (time.perf_counter() - t0) * 1e3
        return total

    leg(False), leg(True)                                  # warm-up
    off, on = [], []
    for _ in range(args.reps):
        off.append(leg(False))
        on.append(leg(True))
    eng.close()
    print(json.dumps(dict(card=card, services=len(gs), ms_off=round(float(np.median(off)), 2),
                          ms_on=round(float(np.median(on)), 2), added_ms=round(float(np.median(on) - np.median(off)), 2),
                          ms_off_all=[round(x, 2) for x in off], ms_on_all=[round(x, 2) for x in on])))


if __name__ == "__main__":
    main()
