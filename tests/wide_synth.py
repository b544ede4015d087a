"""Wide but solvable two-pass services: candidate ranges of 65 to 2048 spans per callee that the exact
window search of the oracle and of the engine still finishes.

A stream of short, non-overlapping requests (one child per callee, nested in DAG order) carries a few
long in-spans.  A long in-span covers `m` consecutive short requests and has `own` children of its own
per callee in the gap before the first of them; `stray` spans per callee start in that gap too but end
after the long in-span (they move the offsets of its later candidates without being feasible for it).
A window is then a star: the long in-span against the short requests it covers.  Counts are balanced
(every callee gets as many children as there are in-spans) by orphan in-spans and filler children at the
end of the stream.

`edges(prob)` measures, with numpy only, what the device paths key on: per in-span and callee the range
length r (spans from lower_bound(start) with start <= end), the offset of the furthest feasible
candidate from lower_bound(start), the E = 1 term-table size 2r, the candidate combinations prod r, and
per 31-in-span redo tile the staged slice of the redo kernel."""
from dataclasses import dataclass, field
from typing import List

import numpy as np

from traceweaver_b200.batch import Problem

SCORE_TILE = 128       # kS3Tile
REDO_TILE = 31         # kWideThreads - 1
NARROW_R = 64          # kS3MaxR: a wider range flags the scoring tile for the redo kernel
WIDE_BITS = 2048       # 32 * kWideW: feasible offsets the redo kernel's maps hold
STAGE_SPANS = 1536     # kStageSpans
TBL_CAP = 3072         # kTblCap
WARP_TBL_CAP = 256     # kWarpTblCap
REDO_COOP = 256        # kRedoCoopCombos
STITCH_COOP = 512      # kStitchCoopCombos
UNIT_MIN = 48          # kStitchUnitMin

# clock -> (request period G, short request length D, timestamp quantum in us)
CLOCKS = {"us": (1000, 300, 1), "ms": (24, 9, 1000)}


@dataclass
class Long:
    pos: int                       # index of the long in-span in the service's start order
    m: int                         # short requests it covers
    own: object = 1                # own children per callee (int or one per callee)
    stray: object = 0              # spans per callee that start inside it and end after it
    inside: bool = False           # start at the first child of the short request before it
    probe: bool = False            # a second in-span right after it (see _probe)


@dataclass
class Case:
    E: int
    longs: List[Long]
    n_short: int
    dag: str = "chain"             # "chain" (callee e after e - 1) or "parallel" (no edges)
    clock: str = "us"
    name: str = ""
    tags: List[str] = field(default_factory=list)


def _per(x, E):
    return list(x) if isinstance(x, (list, tuple)) else [int(x)] * E


def build(case: Case) -> Problem:
    E, (G, D, q) = case.E, CLOCKS[case.clock]
    preds = [[e - 1] if (case.dag == "chain" and e > 0) else [] for e in range(E)]
    ins, kids = [], [[] for _ in range(E)]
    k = max(1, (D - 1) // E)

    def short_kids(t):
        for e in range(E):
            kids[e].append((t + 1 + e * k, t + (e + 1) * k) if case.dag == "chain" else (t + 1, t + D - 1))

    # the short request a long in-span's `pos` lands on: in-spans before it are shorts and earlier longs
    # (a probe counts as one more in-span)
    first = {}
    extra = 0
    for L in sorted(case.longs, key=lambda L: L.pos):
        a = L.pos - extra
        first[id(L)] = a
        extra += 2 if L.probe else 1
    T = lambda j: j * G
    for j in range(case.n_short):
        ins.append((T(j), T(j) + D))
        short_kids(T(j))
    for L in case.longs:
        a = first[id(L)]
        S = T(a - 1) + 1 if L.inside else T(a) - G // 4
        lo = (T(a - 1) + D + 1) if L.inside else S + 1
        hi = T(a) - 1
        end = T(a + L.m - 1) + D + G // 4
        assert T(a + L.m) - G // 4 > end or a + L.m >= case.n_short
        ins.append((S, end))
        own, stray = _per(L.own, E), _per(L.stray, E)
        room = max(1, (hi - lo + 1) // E)
        for e in range(E):
            base = lo + (e * room if case.dag == "chain" else 0)
            span = room if case.dag == "chain" else hi - lo + 1
            for x in range(own[e]):
                s = base + (x % max(1, span // 2))
                kids[e].append((s, min(s + max(0, span // 2 - 1), hi)))
            for x in range(stray[e]):
                s = lo + (x % max(1, hi - lo + 1))
                kids[e].append((s, end + 1 + x))
        if L.probe:
            _probe(case, L, S, end, a, ins, kids)
    prob = _assemble(ins, kids, preds, G, D, q, case.name)
    for L in case.longs:          # every long in-span landed where the case put it
        S = T(first[id(L)] - 1) + 1 if L.inside else T(first[id(L)]) - G // 4
        assert int(prob.in_start[L.pos]) == S * q, (case.name, L.pos)
    return prob


def _assemble(ins, kids, preds, G, D, q, name):
    """The Problem of in-spans `ins` and children `kids` (per callee), in units of q us, with the counts
    balanced: orphan in-spans (no candidates) and filler children after everything else."""
    E = len(kids)
    t_end = max(max(e for _, e in ins), max(e for kk in kids for _, e in kk)) + 10 * G
    need = max(len(kk) for kk in kids) - len(ins)
    for j in range(max(0, need)):
        ins.append((t_end + j * G, t_end + j * G + D))
    t_fill = t_end + (max(0, need) + 2) * G
    for e in range(E):
        for j in range(len(ins) - len(kids[e])):
            kids[e].append((t_fill + 3 * j, t_fill + 3 * j + 1))
    ins.sort(key=lambda x: x[0])
    out_s, out_e = [], []
    for e in range(E):
        kk = sorted(kids[e], key=lambda x: x[0])
        out_s.append(np.array([s for s, _ in kk], np.int64) * q)
        out_e.append(np.array([x for _, x in kk], np.int64) * q)
    a = np.array(ins, np.int64) * q
    prob = Problem(in_start=a[:, 0].copy(), in_end=a[:, 1].copy(), out_start=out_s, out_end=out_e, preds=preds,
                   name=name)
    prob.validate()
    assert prob.in_accelerated_regime()
    return prob


STRONG_Y, STRONG_Q = 51, 52      # in-span indices of strong_cut_case()'s Y and q


def strong_cut_case():
    """A perfect cut next to a wide in-span that only the wide in-span's extent keeps from being strong
    (E = 2, parallel callees, microseconds):
      W = [0, 10000], index 0: candidates c (callee 0, late in W) and w1 (callee 1, early); 70 callee-0
          spans start early in W and end after everything, so W's range is 71 wide and c sits at offset 70;
          one callee-1 span starts before Y and ends after everything
      50 in-spans early in W with no candidates (no cut: W, their prev, ends after them)
      Y = [5000, 10100], index 51: no feasible tuple (no callee-1 child fits), so cut[Y] = 1
      q = [5500, 10200], index 52: its only tuple is (c, z), z a callee-1 child after Y
    W's window takes (c, w1); q, searched under that taken bit, stays unassigned.  The cut at Y is strong
    only if W's extent stops below c: with W's extent [lower_bound(start), upper_bound(end) - 1] it is
    not, the service stays one stitch unit, and q sees c taken."""
    ins = [(0, 10000)] + [(30 + j, 30 + j) for j in range(50)] + [(5000, 10100), (5500, 10200)]
    kids = [[(100 + x, 50000 + x) for x in range(70)] + [(6000, 6100)], [(10, 20), (4000, 50000), (10150, 10190)]]
    return _assemble(ins, kids, [[], []], 1000, 300, 1, "strong-cut")


def _probe(case, L, S, end, a, ins, kids):
    """An E = 1 in-span P right after the long in-span L (its prev is L) whose range stays narrow: 40
    spans start between L and P and end after both (L's range only), then P's own 32 candidates, then L's
    candidates, which P's map holds at offsets 32 and up.  L's tile is redone, P's is not: the cut flag of
    P is k_cut's test of a wide prev against a narrow map, decided by bits 32-63 only."""
    assert case.E == 1 and case.clock == "us"
    G, D, _ = CLOCKS[case.clock]
    p_s, p_e = a * G - 100, end + 100
    for x in range(40):
        kids[0].append((S + 1 + x, p_e + 1 + x))
    for x in range(32):
        kids[0].append((p_s + x, end + 1 + x))
    ins.append((p_s, p_e))


# ---- host-side measurements ---------------------------------------------------------------------------
def feasible_members(prob: Problem, i):
    """Per callee, the sorted original indices that appear in some feasible tuple of in-span i (chains and
    edge-free DAGs: a forward and a backward pass are exact)."""
    E, s, t = prob.E, int(prob.in_start[i]), int(prob.in_end[i])
    cont = [(prob.out_start[e] >= s) & (prob.out_end[e] <= t) for e in range(E)]
    ok = [c.copy() for c in cont]
    for e in range(E):                      # forward: some feasible predecessor child ends before it starts
        for b in prob.preds[e]:
            ends = prob.out_end[b][ok[b]]
            m = ends.min() if len(ends) else np.iinfo(np.int64).max
            ok[e] &= prob.out_start[e] >= m
    for e in reversed(range(E)):            # backward: some feasible successor child starts after it ends
        for f in range(e + 1, E):
            if e in prob.preds[f]:
                st = prob.out_start[f][ok[f]]
                m = st.max() if len(st) else np.iinfo(np.int64).min
                ok[e] &= prob.out_end[e] <= m
    if not all(o.any() for o in ok):
        return [np.zeros(0, np.int64)] * E
    return [np.flatnonzero(o) for o in ok]


def edges(prob: Problem):
    """Per in-span: r [n, E], max feasible offset [n, E] (-1: none), combinations, E = 1 table size; per
    redo tile: its staged slice.  Also which in-spans leave the narrow maps (r > 64 on some callee)."""
    n, E = prob.n_in, prob.E
    lo = np.stack([np.searchsorted(prob.out_start[e], prob.in_start, "left") for e in range(E)], 1)
    up = np.stack([np.searchsorted(prob.out_start[e], prob.in_end, "right") for e in range(E)], 1)
    r = up - lo
    off = np.full((n, E), -1, np.int64)
    for i in np.flatnonzero((r > 0).all(1)):
        for e, mem in enumerate(feasible_members(prob, i)):
            if len(mem):
                off[i, e] = mem[-1] - lo[i, e]
    combos = np.prod(r.astype(np.float64), 1)
    wide = (r > NARROW_R).any(1)
    slices = []
    for i0 in range(0, n, SCORE_TILE):
        for j0 in range(i0, min(i0 + SCORE_TILE, n), REDO_TILE):
            j1 = min(j0 + REDO_TILE, i0 + SCORE_TILE, n)
            me = int(prob.in_end[j0:j1].max())
            tot = sum(int(np.searchsorted(prob.out_start[e], me, "right") -
                          np.searchsorted(prob.out_start[e], prob.in_start[j0], "left")) for e in range(E))
            slices.append((j0, j1, tot, bool(wide[i0:min(i0 + SCORE_TILE, n)].any())))
    tsize = _table_size(prob, r)
    return dict(r=r, off=off, combos=combos, wide=wide, slices=slices, tsize=tsize, lo=lo, up=up)


def _table_size(prob, r):
    tot = np.zeros(prob.n_in, np.int64)
    for e, src in prob.terms():
        tot += r[:, src] * r[:, e] if src >= 0 else r[:, e]
    return tot


def wide_tiles(prob: Problem):
    """Scoring tiles that hold an in-span whose range leaves the narrow maps: the least the redo kernel
    takes (ties and NaN scores can flag more)."""
    w = edges(prob)["wide"]
    return sorted({i // SCORE_TILE for i in np.flatnonzero(w)})


def strong_cuts(prob: Problem, cut, wide_extent=True):
    """k_stitch_units' strong cuts with the maps replaced by the feasible extents (a wide in-span, whose tile
    the redo kernel owns, takes [lower_bound(start), upper_bound(end) - 1] as the kernel does;
    wide_extent=False: [lower_bound(start), lower_bound(start)] instead, to show where that extent decides)."""
    ed = edges(prob)
    n, E = prob.n_in, prob.E
    hi = np.full((n, E), -1, np.int64)
    tiles = set(wide_tiles(prob))
    for i in range(n):
        if i // SCORE_TILE in tiles:
            hi[i] = ed["up"][i] - 1 if wide_extent else ed["lo"][i]
        else:
            hi[i] = np.where(ed["off"][i] >= 0, ed["lo"][i] + ed["off"][i], -1)
    run = np.maximum.accumulate(np.vstack([np.full((1, E), -1), hi[:-1]]), 0)
    strong = (np.asarray(cut[:n]) != 0) & (run < ed["lo"]).all(1)
    strong[0] = False
    return np.flatnonzero(strong)


# ---- the cases --------------------------------------------------------------------------------------
def _e1_longs():
    """E = 1, one long in-span per region, every one in a tile it flags itself (or shares with one that
    does): C = own + stray + m spans in range, the furthest feasible at offset C - 1 - stray."""
    spec = [  # (pos, C)
        (0, 65),      # offset 64, first of a scoring tile
        (128, 66),    # offset 65, first of a scoring tile
        (200, 64),    # offset 63, range 64: narrow itself, in the tile the one at 128 flags; straddles tiles
        (383, 128),   # offset 127, E = 1 table 256 (stitch tables); last of a scoring tile
        (540, 129),   # offset 128, table 258 (stitch lazy path)
        (700, 130),   # offset 129
        (860, 256),   # combinations 256 (redo: per lane); last of a redo tile (768 + 92)
        (1150, 257),  # combinations 257 (redo: whole warp)
        (1450, 1024),  # offset 1023
        (2500, 1025),  # offset 1024
    ]
    return [Long(pos=p, m=c - 1) for p, c in spec]


def cases():
    """name -> Case.  `edge` tags name what a case is there for (checked by check_edges)."""
    C = {}
    C["e1"] = Case(E=1, longs=_e1_longs(), n_short=3560)
    C["e1-c1536"] = Case(E=1, longs=[Long(pos=31, m=1535)], n_short=1701)        # slice 1536, table 3072
    C["e1-c1537"] = Case(E=1, longs=[Long(pos=31, m=1536)], n_short=1701)        # slice 1537, table 3074
    C["e1-off2047"] = Case(E=1, longs=[Long(pos=62, m=2000, stray=47)], n_short=2120)
    C["e1-off2048"] = Case(E=1, longs=[Long(pos=62, m=2000, stray=48)], n_short=2120)
    C["e1-probe"] = Case(E=1, longs=[Long(pos=127, m=24, probe=True)], n_short=400)
    C["e2"] = Case(E=2, longs=[Long(pos=0, m=64), Long(pos=128, m=65), Long(pos=250, m=129),
                               Long(pos=400, m=80), Long(pos=430, m=70, inside=True)], n_short=640)
    C["e3"] = Case(E=3, longs=[Long(pos=93, m=64), Long(pos=300, m=62, stray=[0, 1, 2])], n_short=460)
    C["e5-par"] = Case(E=5, dag="parallel", n_short=300,
                       longs=[Long(pos=0, m=1, own=[65, 0, 0, 0, 0]), Long(pos=40, m=2, own=[2, 2, 2, 2, 0]),
                              Long(pos=80, m=1, own=[8, 18, 2, 0, 0]), Long(pos=160, m=2, own=[4, 4, 4, 4, 0],
                                                                           stray=[70, 0, 0, 0, 0])])
    C["e1-ms"] = Case(E=1, clock="ms", longs=[Long(pos=5, m=70, own=3), Long(pos=127, m=130, own=3)], n_short=400)
    C["e2-ms"] = Case(E=2, clock="ms", longs=[Long(pos=0, m=66, own=3), Long(pos=200, m=64, inside=True)], n_short=330)
    for k, c in C.items():
        c.name = k
    return C
