"""Per-phase cycle shares and path counts of k_stitch in both passes (library built with -DTW_PROFILE_PHASES).
Usage: python scripts/stitch_phase_profile.py [n_services] [hotel|media|alibaba]"""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from traceweaver_b200 import _lib
_lib.SO_PATH = os.path.join(os.path.dirname(_lib.SO_PATH), "libtw_b200_prof.so")
import torch
from traceweaver_b200 import shard
from traceweaver_b200.batch import build_batch_from_blocks
from traceweaver_b200.engine import Engine
S = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
wl = sys.argv[2] if len(sys.argv) > 2 else "hotel"
hb = build_batch_from_blocks(shard.generate_slice(shard.stream_spec(wl, S, 1000, 10), 0, S))
eng = Engine(0); eng.bind(hb); eng.prepare()
p0 = eng.params_pass0(); sc = eng.score(p0, want_used=True); r0 = eng.stitch(p0, sc["cut"], undeleted=sc)
p1 = eng.gmm_refit(*eng.delays(r0["assign"])); top = eng.score(p1, want_used=True)
lib = _lib.load()
buf = (C.c_ulonglong * 16)()
names = ["setup", "run_extent", "run_test", "run_commit", "win_extent", "fast_adopt", "slow_path", "mwis", "win_commit"]
for k, (params, spec) in enumerate(((p0, sc), (p1, top))):
    torch.cuda.synchronize(); lib.tw_debug_stitch_phases(buf, 1)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); eng.stitch(params, sc["cut"], undeleted=spec); b.record(); torch.cuda.synchronize()
    lib.tw_debug_stitch_phases(buf, 1)
    print(f"{wl} {hb.n_problems} services: stitch pass {k} (fast path allowed) {a.elapsed_time(b):.2f} ms")
    tot = sum(buf[:9]) or 1
    print(" ".join(f"{n}={100*buf[q]/tot:.1f}%" for q, n in enumerate(names)))
    print(f"runs={buf[10]} in_spans_in_runs={buf[11]} windows={buf[12]} in_spans_in_windows={buf[13]} "
          f"slow_in_spans={buf[14]} large_mwis_windows={buf[15]}")
    print(f"cycles per service {tot / hb.n_problems:.0f}")
