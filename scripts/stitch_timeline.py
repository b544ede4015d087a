"""Busy warp slots of k_stitch over time in both passes, read from the timeline build of the library:

    python -m traceweaver_b200.csrc.build --timeline
    TW_B200_SO=traceweaver_b200/libtw_b200_timeline.so python scripts/stitch_timeline.py [n_services] [hotel|media|alibaba]

Every warp records the %globaltimer at the start of its first unit and the end of its last one; the
script prints the mean number of busy warps per tenth of the kernel and the share of the kernel's
duration during which fewer than half of the resident warp slots (SMs x 28) are busy."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from traceweaver_b200 import _lib, shard
from traceweaver_b200.batch import build_batch_from_blocks
from traceweaver_b200.engine import Engine

RESIDENT_WARPS_PER_SM = 28      # tw_kernels.cuh: kStitchWarps * kStitchBlocksPerSM
CAP = 1 << 18                   # tw_stitch.cu: kTimelineCap
BINS = 10

lib = _lib.load()
if not hasattr(lib, "tw_debug_stitch_timeline"):
    sys.exit(f"{_lib.SO_PATH} has no stitch timeline: build it with --timeline and name it in TW_B200_SO")
lib.tw_debug_stitch_timeline.argtypes = [C.c_void_p, C.c_int, C.c_int]
S = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
wl = sys.argv[2] if len(sys.argv) > 2 else "hotel"
hb = build_batch_from_blocks(shard.generate_slice(shard.stream_spec(wl, S, 1000, 10), 0, S))
eng = Engine(0); eng.bind(hb); eng.prepare()
p0 = eng.params_pass0(); sc = eng.score(p0, want_used=True); r0 = eng.stitch(p0, sc["cut"], undeleted=sc)
p1 = eng.gmm_refit(*eng.delays(r0["assign"])); top = eng.score(p1, want_used=True)
buf = np.zeros(3 * CAP, np.uint64)
slots = torch.cuda.get_device_properties(0).multi_processor_count * RESIDENT_WARPS_PER_SM


def busy_profile(rec):
    """Piecewise-constant number of busy warps: event times, and the busy count after each event."""
    t = np.concatenate([rec[:, 0], rec[:, 1]]).astype(np.float64)
    d = np.concatenate([np.ones(len(rec)), -np.ones(len(rec))])
    order = np.lexsort((d, t))                     # at equal times the ends come first
    return t[order], np.cumsum(d[order])


for k, (params, spec) in enumerate(((p0, sc), (p1, top))):
    torch.cuda.synchronize()
    assert lib.tw_debug_stitch_timeline(buf.ctypes.data, CAP, 1) == CAP
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); eng.stitch(params, sc["cut"], undeleted=spec); b.record(); torch.cuda.synchronize()
    assert lib.tw_debug_stitch_timeline(buf.ctypes.data, CAP, 1) == CAP
    rec = buf.reshape(CAP, 3)
    rec = rec[rec[:, 1] > 0]
    t, busy = busy_profile(rec)
    t0, t1 = t[0], t[-1]
    dt = np.diff(t)
    below = float(dt[busy[:-1] < slots / 2].sum()) / (t1 - t0)
    integral = np.concatenate([[0.0], np.cumsum(busy[:-1] * dt)])       # piecewise linear in time
    edges = np.linspace(t0, t1, BINS + 1)
    mean_busy = np.diff(np.interp(edges, t, integral)) / np.diff(edges)
    print(f"{wl} {hb.n_problems} services: stitch pass {k} {a.elapsed_time(b):.2f} ms (events), "
          f"warps {len(rec)}, first start to last end {(t1 - t0) / 1e6:.2f} ms, "
          f"peak busy {int(busy.max())} of {slots} slots")
    print("  mean busy warps per tenth: " + " ".join(f"{m:.0f}" for m in mean_busy))
    print(f"  share of the kernel below half of the slots busy: {100 * below:.1f} %")
