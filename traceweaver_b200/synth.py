"""Synthetic span streams of the shapes BASELINE.json names (SURVEY.md §8d): many independent
services, each a stream of incoming requests that fan out to E outgoing endpoints along a fixed
invocation DAG, int64 microsecond timestamps from 1.6e15, n_out == n_in (no skips), ground truth
kept.  Delay/duration laws are log-normal, calibrated on the reference's hotel_reservation traces
(tests/golden fixtures: Poisson arrivals with 33 ms mean inter-arrival at load 100, ~250 us
dispatch gaps, 4-18 ms downstream calls).  Generation is host-side numpy and is NOT part of any
timed region."""
import numpy as np

from .batch import ServiceBlock

T0 = 1_655_760_000_000_000     # us; same epoch range as the Jaeger startTime values

# shape -> (preds, per-ep (gap median us, gap sigma, dur median us, dur sigma), tail median, mode)
SHAPES = {
    # hotel frontend: search -> reservation -> profile, plus the transitive search -> profile edge
    "hotel_frontend": dict(preds=[[], [0], [0, 1]], eps=[(270, 0.6, 15400, 0.45), (195, 0.7, 7300, 1.2),
                                                           (210, 0.6, 4150, 0.55)], tail=(165, 0.7), chain=True),
    # hotel search: geo -> rate
    "hotel_search": dict(preds=[[], [0]], eps=[(267, 0.6, 3700, 0.5), (165, 0.8, 7300, 0.6)], tail=(68, 0.8),
                         chain=True),
    # media nginx: four parallel endpoints, no DAG edges
    "media_nginx": dict(preds=[[], [], [], []], eps=[(250, 0.6, 2500, 0.6), (300, 0.6, 3000, 0.6),
                                                     (350, 0.6, 1500, 0.6), (400, 0.6, 4000, 0.6)],
                        tail=(200, 0.7), chain=False),
    "single": dict(preds=[[]], eps=[(250, 0.6, 5000, 0.6)], tail=(150, 0.7), chain=True),
    # media_microservices as shipped (calibrated on tests/golden/media_load100__*: median / log-sigma of
    # the dispatch gap and of the downstream call per callee, 10 ms mean inter-arrival at load 100).
    # nginx: user / movie-id / unique-id / text in parallel (SURVEY App. B: mean 41, max 2688 tuples)
    "media_nginx_cal": dict(preds=[[], [], [], []], eps=[(393, 0.49, 3516, 0.67), (524, 0.50, 6438, 0.64),
                                                         (668, 0.41, 3000, 0.73), (588, 0.43, 3044, 0.72)],
                            tail=(2629, 0.6), chain=False, ia100=10_000.0),
    # movie-id-service: rating and compose-review in parallel
    "media_movie_id": dict(preds=[[], []], eps=[(1000, 0.45, 2981, 0.80), (1320, 0.59, 1498, 0.96)],
                           tail=(394, 0.7), chain=False, ia100=10_000.0),
    # user / rating / unique-id / text-service: one call to compose-review
    "media_leaf": dict(preds=[[]], eps=[(600, 0.85, 1700, 0.95)], tail=(150, 0.8), chain=True, ia100=10_000.0),
    # alibaba-shaped call graphs (the trace itself is an LFS pointer in the reference; schema
    # alibaba-analysis/real-parser.py:308-359: millisecond rpc timestamps x1000).  Depth-2 fan-outs
    # of 1..4 downstream calls, sequential or parallel.
    "ali_chain4": dict(preds=[[], [0], [1], [2]], eps=[(1000, 0.8, 4000, 0.9)] * 4, tail=(1000, 0.8), chain=True,
                       ia100=10_000.0),
    "ali_par3": dict(preds=[[], [], []], eps=[(1000, 0.8, 5000, 0.9), (2000, 0.8, 3000, 0.9), (1500, 0.8, 8000, 0.9)],
                     tail=(1000, 0.8), chain=False, ia100=10_000.0),
    "ali_chain2": dict(preds=[[], [0]], eps=[(1000, 0.8, 6000, 0.9), (1000, 0.8, 3000, 0.9)], tail=(1000, 0.8),
                       chain=True, ia100=10_000.0),
    "ali_leaf": dict(preds=[[]], eps=[(1000, 0.9, 5000, 1.0)], tail=(1000, 0.8), chain=True, ia100=10_000.0),
}
INTERARRIVAL_US_AT_LOAD_100 = 33_300.0


ALIBABA_MAX_LOAD = 50.0
MAX_CALL_US = 150_000   # downstream calls time out: the reference's hotel traces top out near 150 ms


def _lognormal(rng, median, sigma, shape, floor=1):
    v = rng.lognormal(np.log(median), sigma, size=shape)
    return np.clip(np.rint(v), floor, MAX_CALL_US).astype(np.int64)


def make_block(shape: str, n_services: int, n_in: int = 1000, load: float = 100.0, seed: int = 10,
               quantum_us: int = 1) -> ServiceBlock:
    """quantum_us > 1 rounds every timestamp down to that grid (1000: millisecond clocks, as in the
    Alibaba trace) — equal timestamps, zero-length gaps and exact score ties become common."""
    spec = SHAPES[shape]
    rng = np.random.default_rng(seed)
    S, n = n_services, n_in
    E = len(spec["eps"])
    ia100 = spec.get("ia100", INTERARRIVAL_US_AT_LOAD_100)
    ia = np.maximum(np.rint(rng.exponential(ia100 * 100.0 / load, size=(S, n))), 1).astype(np.int64)
    in_start = T0 + np.cumsum(ia, axis=1)
    t = in_start.copy()
    latest = in_start.copy()
    starts, ends = [], []
    for e, (gm, gs, dm, ds) in enumerate(spec["eps"]):
        base = t if spec["chain"] else in_start
        s = base + _lognormal(rng, gm, gs, (S, n))
        en = s + _lognormal(rng, dm, ds, (S, n))
        starts.append(s)
        ends.append(en)
        t = en
        latest = np.maximum(latest, en)
    in_end = latest + _lognormal(rng, spec["tail"][0], spec["tail"][1], (S, n))
    if quantum_us > 1:
        q = quantum_us
        in_start, in_end = in_start // q * q, in_end // q * q
        starts = [s // q * q for s in starts]
        ends = [e // q * q for e in ends]
        order = np.argsort(in_start, axis=1, kind="stable")      # (start, end) order after rounding
        tie_rows = np.flatnonzero((np.diff(in_start, axis=1) == 0).any(axis=1))
        for r in tie_rows:
            order[r] = np.lexsort((in_end[r], in_start[r]))
        in_start = np.take_along_axis(in_start, order, axis=1)
        in_end = np.take_along_axis(in_end, order, axis=1)
        starts = [np.take_along_axis(s, order, axis=1) for s in starts]
        ends = [np.take_along_axis(e, order, axis=1) for e in ends]
    out_start, out_end, truth = [], [], np.empty((E, S, n), np.int32)
    rows = np.arange(S)[:, None]
    for e in range(E):
        order = np.argsort(starts[e], axis=1, kind="stable")
        s_sorted = np.take_along_axis(starts[e], order, axis=1)
        e_sorted = np.take_along_axis(ends[e], order, axis=1)
        tie_rows = np.flatnonzero((np.diff(s_sorted, axis=1) == 0).any(axis=1))
        for r in tie_rows:        # (start, end) order where starts tie (executor.py:1111-1112)
            o2 = np.lexsort((ends[e][r], starts[e][r]))
            order[r] = o2
            s_sorted[r] = starts[e][r][o2]
            e_sorted[r] = ends[e][r][o2]
        inv = np.empty_like(order)
        inv[rows, order] = np.arange(n)[None, :]
        out_start.append(np.ascontiguousarray(s_sorted))
        out_end.append(np.ascontiguousarray(e_sorted))
        truth[e] = inv
    return ServiceBlock(in_start=np.ascontiguousarray(in_start), in_end=np.ascontiguousarray(in_end),
                        out_start=out_start, out_end=out_end, preds=spec["preds"], truth=truth,
                        name=f"{shape}@load{load:g}")


def hotel_stream(n_services: int, n_in: int = 1000, loads=(25, 50, 75, 100, 125, 150), seed: int = 10):
    """hotel_reservation-shaped stream: alternating `frontend` (E=3) and `search` (E=2) services over
    the six load levels of the reference's dataset directories."""
    blocks = []
    per = max(1, n_services // (2 * len(loads)))
    k = 0
    for li, load in enumerate(loads):
        for shape in ("hotel_frontend", "hotel_search"):
            cnt = per if (li, shape) != (len(loads) - 1, "hotel_search") else max(1, n_services - per * (2 * len(loads) - 1))
            blocks.append(make_block(shape, cnt, n_in, load, seed + k))
            k += 1
    return blocks


def media_stream(n_services: int, n_in: int = 1000, loads=(25, 50, 75, 100, 125, 150), seed: int = 10):
    """media_microservices-shaped stream (BASELINE configs[2]): per trace directory the reference
    solves nginx (E=4 parallel), movie-id-service (E=2 parallel) and four one-callee services; six
    load levels like the shipped directories."""
    mix = (("media_nginx_cal", 1), ("media_movie_id", 1), ("media_leaf", 4))
    per_unit = max(1, n_services // (6 * len(loads)))
    blocks, k = [], 0
    for load in loads:
        for shape, mult in mix:
            blocks.append(make_block(shape, per_unit * mult, n_in, load, seed + k))
            k += 1
    return blocks


def alibaba_stream(n_services: int = 2000, n_in: int = 1250, compress=(1, 200, 1000, 4000, 10000, 15000),
                   seed: int = 10, quantum_us: int = 1000):
    """alibaba-shaped window (BASELINE configs[3]; synthetic — the trace is not shipped): services
    with 1..4 downstream calls, millisecond clocks, time compression as in exps/exp5
    (helpers/transforms.py:10-40 divides arrival times by the factor; executor.py:1091 caps it by the
    replica count, drawn here as 2^k <= 4096): the effective load is what the generator's `load` is."""
    shapes = ("ali_leaf", "ali_chain2", "ali_par3", "ali_chain4", "ali_leaf", "ali_chain2")
    rng = np.random.default_rng(seed)
    per = max(1, n_services // (len(shapes) * len(compress)))
    blocks, k = [], 0
    for cf in compress:
        for shape in shapes:
            replicas = 2 ** int(rng.integers(0, 13))
            factor = max(1, int(np.ceil(cf / replicas)))
            # an uncompressed service sees ~1 request per second; load 100 = one per 10 ms.  The generator
            # stops at load 50: with millisecond clocks the three-callee parallel shape at load 100 has
            # 30-in-span windows of interchangeable candidates; the engine's search (priced bound,
            # tw_core.cuh) finishes them in ~2e5 nodes, but the ORACLE's plain branch and bound — the
            # checker of every bench leg — exceeds its 20 M-node budget there
            load = min(1.0 * factor, ALIBABA_MAX_LOAD)
            blocks.append(make_block(shape, per, n_in, load, seed + k, quantum_us=quantum_us))
            k += 1
    return blocks


def _sort_rows(start, end):
    """Rows sorted by (start, end): sorted copies and rank[s, r] = position of element r in row s."""
    order = np.lexsort((end, start), axis=-1)
    rank = np.empty_like(order)
    np.put_along_axis(rank, order, np.arange(order.shape[1])[None, :], axis=1)
    return np.take_along_axis(start, order, axis=1), np.take_along_axis(end, order, axis=1), rank


def hotel_tree(n_replicas: int, n_req: int = 1000, load: float = 100.0, seed: int = 10):
    """Requests of a two-tier hotel_reservation-shaped deployment, for the request trees (traces.py).  Each of
    `n_replicas` replicas gets `n_req` requests at its frontend, which calls search, then reservation, then
    profile (the hotel_frontend DAG); search calls geo, then rate (hotel_search).  Frontend and search are the
    solved services; every server span lies inside its client span (a network hop of a few tens of us each
    way).  Returns dict(blocks=[frontend, search] ServiceBlocks, hb (frontend problems, then search problems),
    in_caller: int32 [n_in] node ids as traces.caller_links gives them, truth: the true assignment,
    in_request: int32 [n_in] the request every in-span serves, numbered replica * n_req + arrival)."""
    rng = np.random.default_rng(seed)
    S, n = n_replicas, n_req
    lat = lambda: _lognormal(rng, 40, 0.5, (S, n))
    ia = np.maximum(np.rint(rng.exponential(INTERARRIVAL_US_AT_LOAD_100 * 100.0 / load, size=(S, n))), 1).astype(np.int64)
    f_start = T0 + np.cumsum(ia, axis=1)
    c0s = f_start + _lognormal(rng, 270, 0.6, (S, n))                 # frontend -> search (client)
    s_start = c0s + lat()                                               # search (server)
    geo_s = s_start + _lognormal(rng, 267, 0.6, (S, n))
    geo_e = geo_s + _lognormal(rng, 3700, 0.5, (S, n))
    rate_s = geo_e + _lognormal(rng, 165, 0.8, (S, n))
    rate_e = rate_s + _lognormal(rng, 7300, 0.6, (S, n))
    s_end = rate_e + _lognormal(rng, 68, 0.8, (S, n))
    c0e = s_end + lat()
    res_s = c0e + _lognormal(rng, 195, 0.7, (S, n))
    res_e = res_s + _lognormal(rng, 7300, 1.2, (S, n))
    pro_s = res_e + _lognormal(rng, 210, 0.6, (S, n))
    pro_e = pro_s + _lognormal(rng, 4150, 0.55, (S, n))
    f_end = pro_e + _lognormal(rng, 165, 0.7, (S, n))

    def block(in_s, in_e, calls, preds, name):
        in_s, in_e, in_rank = _sort_rows(in_s, in_e)
        out_s, out_e, ranks = [], [], []
        truth = np.empty((len(calls), S, n), np.int32)
        for e, (cs, ce) in enumerate(calls):
            a, b, rk = _sort_rows(cs, ce)
            out_s.append(a)
            out_e.append(b)
            ranks.append(rk)
            np.put_along_axis(truth[e], in_rank, rk, axis=1)             # in-span of request r -> its call
        return ServiceBlock(in_start=in_s, in_end=in_e, out_start=out_s, out_end=out_e, preds=preds, truth=truth,
                            name=name), in_rank, ranks

    front, _, f_ranks = block(f_start, f_end, [(c0s, c0e), (res_s, res_e), (pro_s, pro_e)], [[], [0], [0, 1]],
                              f"hotel_tree_frontend@load{load:g}")
    search, s_rank, _ = block(s_start, s_end, [(geo_s, geo_e), (rate_s, rate_e)], [[], [0]],
                              f"hotel_tree_search@load{load:g}")
    from .batch import build_batch_from_blocks
    hb = build_batch_from_blocks([front, search])
    n_in = 2 * S * n
    rows = np.arange(S)[:, None]
    in_caller = np.empty((S, n), np.int32)
    # search in-span of request r (node S*n + s*n + rank) <- the frontend's call to search (ep 0 of problem s)
    in_caller[rows, s_rank] = n_in + (rows * 3) * n + f_ranks[0]
    in_caller = np.concatenate([np.full(S * n, -1, np.int32), in_caller.reshape(-1)])
    request = (rows * n + np.arange(n)[None, :]).astype(np.int32)      # request number of (replica, arrival)
    in_request = np.empty((2, S, n), np.int32)
    in_request[0] = request                                             # frontend arrivals are in start order
    in_request[1][rows, s_rank] = request
    return dict(blocks=[front, search], hb=hb, in_caller=in_caller, truth=truth_assign([front, search]),
                in_request=in_request.reshape(-1))


def span_count(blocks):
    return int(sum(b.in_start.size * (1 + len(b.out_start)) for b in blocks))


def truth_assign(blocks):
    """Ground-truth assignment array in the engine's layout (assign[tuple_off[p] + e*n + i])."""
    return np.concatenate([np.transpose(b.truth, (1, 0, 2)).reshape(-1) for b in blocks]).astype(np.int32)
