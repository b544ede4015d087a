"""Per-phase device time of the path on a synthetic hotel-shaped stream (CUDA events).
Usage: python scripts/time_phases.py [n_services] [n_in]"""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from traceweaver_b200 import synth
from traceweaver_b200.batch import build_batch_from_blocks
from traceweaver_b200.engine import Engine

S = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
n_in = int(sys.argv[2]) if len(sys.argv) > 2 else 1000
wl = sys.argv[3] if len(sys.argv) > 3 else None          # "media" / "alibaba" / "hotel": bench.py's streams
t0 = time.time()
if wl:
    from traceweaver_b200 import shard
    blocks = shard.generate_slice(shard.stream_spec(wl, S, n_in, 10), 0, S)
else:
    blocks = synth.hotel_stream(S, n_in, seed=10)
hb = build_batch_from_blocks(blocks)
nsp = synth.span_count(blocks); print(f"{hb.n_problems} services, {nsp/1e6:.2f} M spans, gen {time.time()-t0:.1f}s")
eng = Engine(0)
t0 = time.time(); eng.bind(hb); torch.cuda.synchronize(); print(f"bind+upload {time.time()-t0:.3f}s")
truth = torch.from_numpy(synth.truth_assign(blocks)).cuda()

def timed(name, fn, reps=3):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); out = fn(); b.record(); torch.cuda.synchronize(); ts.append(a.elapsed_time(b))
    print(f"  {name:28s} {min(ts):9.3f} ms   {nsp/min(ts)/1e3:9.1f} M spans/s")
    return out

timed("prepare (prev+sort)", eng.prepare)
p0 = timed("params_pass0", eng.params_pass0)
timed("score (windows only)", eng.score)
sc = timed("score (gauss, topk+used)", lambda: eng.score(p0, want_used=True))
timed("stitch pass0 slow path", lambda: eng.stitch(p0, sc["cut"]))
r0 = timed("stitch pass0 fast path", lambda: eng.stitch(p0, sc["cut"], undeleted=sc))
dc = timed("delays", lambda: eng.delays(r0["assign"]))
p1 = timed("gmm_refit", lambda: eng.gmm_refit(dc[0], dc[1]))
top = timed("score (gmm, topk+used)", lambda: eng.score(p1, want_used=True))
timed("stitch pass1 slow path", lambda: eng.stitch(p1, sc["cut"]))
r1 = timed("stitch pass1 fast path", lambda: eng.stitch(p1, sc["cut"], undeleted=top))
eng.status()
from traceweaver_b200.predictor import solve_bound
timed("whole path (resident)", lambda: solve_bound(eng))
a = r1["assign"]; ok = (a == truth)
# per in-span accuracy needs all eps: reduce per problem
acc = []
for p in range(0, hb.n_problems, max(1, hb.n_problems // 64)):
    to, n = int(hb.prob_tuple_off[p]), int(hb.prob_in_off[p+1]-hb.prob_in_off[p]); E = int(hb.prob_ep_off[p+1]-hb.prob_ep_off[p])
    acc.append(ok[to:to+n*E].reshape(E, n).all(dim=0).float().mean().item())
c = r1["counters"].cpu().numpy()
print(f"accuracy (sampled services) mean {np.mean(acc):.4f}; unassigned {c[:,1].sum()}; max mwis nodes {c[:,2].max()}; status {c[:,3].min()}")
nf = sc["n_feasible"].float(); print(f"feasible tuples/in-span mean {nf.mean().item():.2f} max {nf.max().item():.0f}")
