"""Per-phase cycle shares and work counters of one kernel, read from the phase counters of the profiling
build of the library:

    python -m traceweaver_b200.csrc.build --prof
    TW_B200_SO=traceweaver_b200/libtw_b200_prof.so python scripts/phase_profile.py {score|stitch|gmm} [n_services] [workload]

score: k_score3 in the pass-0 call (windows + top-K) and the mixture call (top-K only); stitch: k_stitch
in both passes; gmm: the fit kernels of one refit.  workload: hotel (default), media or alibaba, the
streams bench.py runs.  The slots of each kernel's counters are listed where the kernel file declares
them (tw_score3.cu, tw_stitch.cu, tw_gmm.cu)."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from traceweaver_b200 import _lib, shard
from traceweaver_b200.batch import build_batch_from_blocks
from traceweaver_b200.engine import Engine
from traceweaver_b200.predictor import solve_bound

KERNELS = ("score", "stitch", "gmm")           # in the order of tw_debug_phases' kernel argument
if len(sys.argv) < 2 or sys.argv[1] not in KERNELS:
    sys.exit(__doc__)
kernel = sys.argv[1]
S = int(sys.argv[2]) if len(sys.argv) > 2 else 4096
wl = sys.argv[3] if len(sys.argv) > 3 else "hotel"
lib = _lib.load()
if not hasattr(lib, "tw_debug_phases"):
    sys.exit(f"{_lib.SO_PATH} has no phase counters: build it with --prof and name it in TW_B200_SO")
lib.tw_debug_phases.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int]
buf = (C.c_ulonglong * 24)()                  # kPhaseSlots (tw_kernels.cuh)
hb = build_batch_from_blocks(shard.generate_slice(shard.stream_spec(wl, S, 1000, 10), 0, S))
eng = Engine(0); eng.bind(hb)


def counters():
    """The kernel's counters since the last call, read once the device is idle, and zeroed."""
    torch.cuda.synchronize()
    rc = lib.tw_debug_phases(KERNELS.index(kernel), buf, len(buf), 1)
    assert rc == 0, rc
    return list(buf)


def first_pass():
    eng.prepare()
    p0 = eng.params_pass0(); sc = eng.score(p0, want_used=True); r0 = eng.stitch(p0, sc["cut"], undeleted=sc)
    return p0, sc, eng.delays(r0["assign"])


def profile_score():
    res = solve_bound(eng)
    names = ["setup+staging", "ranges", "admission/rest", "term tables", "2a feasibility", "2b scores", "2c top-K", "results"]
    n_in = int(hb.prob_in_off[-1])
    for label, prm in (("gauss pass (windows + top-K)", None), ("mixture pass (top-K only)", res["params_pass1"])):
        counters()
        if prm is None:
            p0 = eng.params_pass0(); eng.score(p0, want_used=True)
        else:
            eng.score(prm, out=dict(cut=res["cut"]), keep_windows=True)
        c = counters()
        tot = sum(c[:8]) or 1
        print(label)
        print("  " + " ".join(f"{n}={100*c[k]/tot:.1f}%" for k, n in enumerate(names)))
        rounds = max(c[12], 1)
        print(f"  per in-span: slots {c[10]/n_in:.2f} (valid {c[14]/n_in:.2f}) combos {c[11]/n_in:.2f} feasible {c[13]/n_in:.2f}; "
              f"rounds per warp-tile {rounds/ (n_in/32):.2f}; warp cycles per in-span {tot/n_in:.0f}")
        print(f"  tiles flagged for the sequential kernel: staging overflow {c[15]}, range/combination limits {c[16]} warps, "
              f"ties/NaN {c[17]} warps; tiles {eng.tile_count()}")


def profile_stitch():
    p0, sc, dc = first_pass()
    p1 = eng.gmm_refit(*dc); top = eng.score(p1, want_used=True)
    names = ["setup", "run_extent", "run_test", "run_commit", "win_extent", "fast_adopt", "slow_path", "mwis", "win_commit"]
    for k, (params, spec) in enumerate(((p0, sc), (p1, top))):
        counters()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); eng.stitch(params, sc["cut"], undeleted=spec); b.record()
        c = counters()
        print(f"{wl} {hb.n_problems} services: stitch pass {k} (fast path allowed) {a.elapsed_time(b):.2f} ms")
        tot = sum(c[:9]) or 1
        print(" ".join(f"{n}={100*c[q]/tot:.1f}%" for q, n in enumerate(names)))
        print(f"runs={c[10]} in_spans_in_runs={c[11]} windows={c[12]} in_spans_in_windows={c[13]} "
              f"slow_in_spans={c[14]} large_mwis_windows={c[15]}")
        print(f"cycles per service {tot / hb.n_problems:.0f}")


def profile_gmm():
    _, _, dc = first_pass()
    eng.gmm_refit(*dc)
    counters()
    eng.gmm_refit(*dc)
    c = counters()
    names = ["seeding", "lloyd", "init_mstep", "em", "score"]
    tot = sum(c[:5]) or 1
    print(" ".join(f"{n}={100*c[k]/tot:.1f}%" for k, n in enumerate(names)))
    print(f"fits={c[7]} lloyd_iters/fit={c[5]/max(c[7],1):.1f} em_iters/fit={c[6]/max(c[7],1):.1f}")


{"score": profile_score, "stitch": profile_stitch, "gmm": profile_gmm}[kernel]()
