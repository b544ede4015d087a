"""Float64 microsecond inputs for the tests of the fractional-timestamp path (tw_engine_bind_f64).

executor.py --compress_factor CF (transforms.repeat_change_spans) divides every span's start time by CF
and keeps its duration, so a span reaches FindAssignments with start = start_us / CF (a float) and
end = start + duration in float arithmetic."""
import math

import numpy as np

from traceweaver_b200.batch import Problem

FIXED_BITS = 55


def compress(prob: Problem, cf) -> Problem:
    """The problem as the reference sees it after --compress_factor cf (float64 times)."""
    def f(start, end):
        s = np.asarray(start, np.int64).astype(np.float64) / float(cf)
        return s, s + (np.asarray(end, np.int64) - np.asarray(start, np.int64)).astype(np.float64)
    in_s, in_e = f(prob.in_start, prob.in_end)
    outs = [f(s, e) for s, e in zip(prob.out_start, prob.out_end)]
    return Problem(in_start=in_s, in_end=in_e, out_start=[o[0] for o in outs], out_end=[o[1] for o in outs],
                   preds=prob.preds, name=f"{prob.name}/cf{cf}")


def times(prob: Problem):
    return [prob.in_start, prob.in_end] + list(prob.out_start) + list(prob.out_end)


def shift_rule(values):
    """s_p of the engine: the smallest s >= 0 with x * 2^s an integer for every x (None: NaN / inf /
    max|x| * 2^s >= 2^55, the inputs the engine rejects)."""
    s, top = 0, 0.0
    for x in values:
        x = float(x)
        if not math.isfinite(x):
            return None
        den = x.as_integer_ratio()[1]               # a power of two
        s = max(s, den.bit_length() - 1)
        top = max(top, abs(x))
    return None if math.ldexp(top, s) >= 2.0 ** FIXED_BITS else s


def reference_sums_exact(prob: Problem):
    """True iff every difference the reference forms between two times of the problem is exact (they all
    lie within a factor of two of each other: Sterbenz) and every pass-0 batch sum (sorted arrays,
    100-span batches and their tenths, V3:590-617) is exact when summed left to right in doubles."""
    v = np.concatenate([np.asarray(a, np.float64) for a in times(prob)])
    lo, hi = float(np.abs(v).min()), float(np.abs(v).max())
    if not (np.all(v > 0) and hi <= 2 * lo):
        return False
    n = prob.n_in
    ins, ine = np.sort(prob.in_start), np.sort(prob.in_end)
    pairs = []
    for e, src in prob.terms():
        os_, oe = np.sort(prob.out_start[e]), np.sort(prob.out_end[e])
        if src >= 0:
            pairs.append((np.sort(prob.out_end[src]), os_))
        elif src == -1:
            pairs.append((ins, os_))
        else:
            pairs.append((oe, ine))
    sh = shift_rule(v)
    fx = lambda a: [int(math.ldexp(float(x), sh)) for x in a]       # exact integers X = x * 2^s
    for t1, t2 in pairs:
        X1, X2 = fx(t1), fx(t2)
        for s in range(0, n, 100):
            z = min(n, s + 100)
            m = z - s
            bs = (m + 9) // 10
            ranges = [(s, z)] + [(s + q * bs, min(z, s + (q + 1) * bs)) for q in range(10) if q * bs < m]
            for a, b in ranges:
                acc = 0.0
                for j in range(a, b):
                    acc += float(t2[j]) - float(t1[j])
                if math.ldexp(acc, sh) != sum(X2[a:b]) - sum(X1[a:b]):
                    return False
    return True
# (fixture, factor) pairs whose compressed instances the oracle's plain branch and bound solves within its
# 20 M-node budget in seconds: compression packs more requests into every window (durations are kept), and
# at factors 200 and 15000 many services' windows become intractable for it
SOLVABLE = {
    3: (
        "alibaba_synth__S0",
        "alibaba_synth__S1",
        "alibaba_synth__S2",
        "alibaba_synth__kCbekANd0f0RpzKC-loop",
        "hotel_load100__frontend",
        "hotel_load100__search",
        "hotel_load125__frontend",
        "hotel_load125__search",
        "hotel_load150__frontend",
        "hotel_load150__search",
        "hotel_load25__frontend",
        "hotel_load25__search",
        "hotel_load50__frontend",
        "hotel_load50__search",
        "hotel_load75__frontend",
        "hotel_load75__search",
        "media_load100__movie-id-service",
        "media_load100__rating-service",
        "media_load100__text-service",
        "media_load100__unique-id-service",
        "media_load100__user-service",
        "media_load125__movie-id-service",
        "media_load125__nginx",
        "media_load125__rating-service",
        "media_load125__text-service",
        "media_load125__unique-id-service",
        "media_load125__user-service",
        "media_load150__movie-id-service",
        "media_load150__rating-service",
        "media_load150__text-service",
        "media_load150__unique-id-service",
        "media_load150__user-service",
        "media_load25__movie-id-service",
        "media_load25__nginx",
        "media_load25__rating-service",
        "media_load25__text-service",
        "media_load25__unique-id-service",
        "media_load25__user-service",
        "media_load50__movie-id-service",
        "media_load50__nginx",
        "media_load50__rating-service",
        "media_load50__text-service",
        "media_load50__unique-id-service",
        "media_load50__user-service",
        "media_load75__movie-id-service",
        "media_load75__nginx",
        "media_load75__rating-service",
        "media_load75__text-service",
        "media_load75__unique-id-service",
        "media_load75__user-service",
        "node_load100__init-service",
        "node_load100__service1",
        "node_load100__service2",
        "node_load100__service3",
        "node_load125__init-service",
        "node_load125__service1",
        "node_load125__service2",
        "node_load125__service3",
        "node_load150__init-service",
        "node_load150__service1",
        "node_load150__service2",
        "node_load150__service3",
        "node_load25__init-service",
        "node_load25__service1",
        "node_load25__service2",
        "node_load25__service3",
        "node_load50__init-service",
        "node_load50__service1",
        "node_load50__service2",
        "node_load50__service3",
        "node_load75__init-service",
        "node_load75__service1",
        "node_load75__service2",
        "node_load75__service3",
    ),
    200: (
        "alibaba_synth__S1",
        "alibaba_synth__S2",
        "alibaba_synth__kCbekANd0f0RpzKC-loop",
        "media_load100__rating-service",
        "media_load25__movie-id-service",
        "media_load25__rating-service",
        "media_load25__text-service",
        "media_load25__unique-id-service",
        "media_load25__user-service",
        "media_load50__rating-service",
        "media_load50__text-service",
        "media_load50__unique-id-service",
        "media_load50__user-service",
        "media_load75__text-service",
        "media_load75__unique-id-service",
        "media_load75__user-service",
        "node_load100__init-service",
        "node_load100__service1",
        "node_load100__service2",
        "node_load100__service3",
        "node_load125__init-service",
        "node_load125__service2",
        "node_load25__init-service",
        "node_load25__service1",
        "node_load25__service2",
        "node_load25__service3",
        "node_load50__init-service",
        "node_load50__service1",
        "node_load50__service2",
        "node_load75__init-service",
        "node_load75__service1",
        "node_load75__service2",
    ),
    15000: (
        "alibaba_synth__S0",
        "alibaba_synth__S1",
        "alibaba_synth__S2",
        "alibaba_synth__kCbekANd0f0RpzKC-loop",
        "media_load25__rating-service",
        "media_load25__text-service",
        "media_load25__unique-id-service",
        "media_load25__user-service",
        "media_load50__text-service",
        "media_load50__unique-id-service",
        "media_load50__user-service",
        "media_load75__text-service",
        "media_load75__user-service",
        "node_load100__init-service",
        "node_load100__service3",
        "node_load125__init-service",
        "node_load25__init-service",
        "node_load50__init-service",
        "node_load50__service2",
        "node_load50__service3",
        "node_load75__init-service",
    ),
}
