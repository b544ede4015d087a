"""Time only the refit, of the library TW_B200_SO names (default: the in-tree build)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from traceweaver_b200 import _lib, synth
from traceweaver_b200.batch import build_batch_from_blocks
from traceweaver_b200.engine import Engine
blocks = synth.hotel_stream(8192, 1000, seed=10); hb = build_batch_from_blocks(blocks)
eng = Engine(0); eng.bind(hb); eng.prepare()
p0 = eng.params_pass0(); sc = eng.score(p0, want_used=True); r0 = eng.stitch(p0, sc["cut"], undeleted=sc)
d, c = eng.delays(r0["assign"])
for _ in range(2): eng.gmm_refit(d, c)
torch.cuda.synchronize()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for _ in range(3): eng.gmm_refit(d, c)
b.record(); torch.cuda.synchronize()
print(_lib.SO_PATH, "gmm_refit ms", a.elapsed_time(b) / 3)
