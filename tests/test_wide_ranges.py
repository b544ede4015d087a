"""The stepped device code (tests/emul) against the oracle on services whose candidate ranges leave the
64-bit maps of the scoring kernel (tests/wide_synth.py): ranges of 65 to 2048 spans, the redo kernel's
staged and unstaged slices, its term-table cap and whole-warp combinations, the stitch's lazy and
whole-warp tiers on wide ranges, a wide prev across a scoring-tile boundary, and a long in-span searched
under bits taken by earlier windows.  Indices exactly, scores bit-equal.  CPU only."""
from functools import lru_cache, partial

import numpy as np
import pytest

import wide_synth as ws
from emul_backend import EmulBatch
from oracle import tw_oracle
from traceweaver_b200 import _abi
from traceweaver_b200.batch import build_batch

CASES = ws.cases()
SOLVED = [k for k in CASES if k != "e1-off2048"]
BACKENDS = {"emul": EmulBatch, "emul-lazy": partial(EmulBatch, table_cap=0),
            "emul-combos": partial(EmulBatch, light_combos=0)}


@lru_cache(maxsize=None)
def problem(name):
    return ws.build(CASES[name])


@lru_cache(maxsize=None)
def oracle_run(name):
    """Every pass of the oracle: pass-0 Gaussians, score and stitch, the refit on the stitch's delays,
    pass-1 score and stitch under those mixtures."""
    prob = problem(name)
    hb = build_batch([prob])
    ob = tw_oracle.OracleBatch(hb)
    g = ob.params_pass0()
    sc = ob.score(gauss=g)
    st = ob.stitch(sc["cut"], gauss=g)
    d, c = ob.delays(st["assign"])
    mix, _, _ = tw_oracle.gmm_refit(hb.term_sample_off, d, c, seed_select=10)
    return dict(prob=prob, hb=hb, gauss=g, sc=sc, st=st, mix=mix, sc1=ob.score(mix=mix),
                st1=ob.stitch(sc["cut"], mix=mix))


def edge_table():
    """edge -> [cases that reach it], measured on the generated arrays (numpy only)."""
    hit = {}

    def add(edge, name):
        hit.setdefault(edge, set()).add(name)

    for name, case in CASES.items():
        prob = problem(name)
        ed = ws.edges(prob)
        off = ed["off"]
        for v in (63, 64, 65, 127, 128, 129, 1023, 1024, 2047, 2048):
            if (off.max(1) == v).any():
                add(f"offset {v}", name)
        wide = ed["wide"]
        for j0, j1, tot, flagged in ed["slices"]:
            if flagged and tot in (ws.STAGE_SPANS, ws.STAGE_SPANS + 1):
                add(f"slice {tot}", name)
        if prob.E == 1:
            for t in (256, 258, 3072, 3074):
                if (wide_in_flagged(prob, ed) & (ed["tsize"] == t)).any():
                    add(f"E=1 table {t}", name)
        fl = wide_in_flagged(prob, ed)
        for P in (256, 257, 512, 513):
            if (fl & (ed["combos"] == P)).any():
                add(f"combinations {P}", name)
        # a long in-span as prev of the first in-span of the next scoring tile, that tile not flagged
        tiles = set(ws.wide_tiles(prob))
        prev = np.concatenate([[0], np.maximum.accumulate(prob.in_end)[:-1]])
        for i0 in range(ws.SCORE_TILE, prob.n_in, ws.SCORE_TILE):
            pi = int(np.flatnonzero(prob.in_end[:i0] == prev[i0])[-1])
            if wide[pi] and i0 // ws.SCORE_TILE not in tiles and (i0 - 1) // ws.SCORE_TILE in tiles and pi == i0 - 1:
                add("wide prev of a tile's first in-span, tile not redone", name)
        # a long in-span whose first candidates were taken by an earlier window: it starts inside the
        # short request before it (at that request's first child) and opens a window at the size cap
        for L in case.longs:
            if L.inside:
                add("long in-span searched under taken bits", name)
    return hit


def wide_in_flagged(prob, ed):
    """in-spans of the scoring tiles the redo kernel takes (at least those: a range over 64)"""
    tiles = set(ws.wide_tiles(prob))
    return np.array([i // ws.SCORE_TILE in tiles for i in range(prob.n_in)])


EDGES = ["offset 63", "offset 64", "offset 65", "offset 127", "offset 128", "offset 129", "offset 1023",
         "offset 1024", "offset 2047", "offset 2048", "slice 1536", "slice 1537", "E=1 table 256",
         "E=1 table 258", "E=1 table 3072", "E=1 table 3074", "combinations 256", "combinations 257",
         "combinations 512", "combinations 513", "wide prev of a tile's first in-span, tile not redone",
         "long in-span searched under taken bits", "strong cut before and after a long in-span",
         "cut kept from being strong by a wide in-span's extent alone"]


def test_every_edge_is_reached():
    hit = edge_table()
    for name in SOLVED:                      # strong cuts need the oracle's cut flags
        prob, cut = problem(name), oracle_run(name)["sc"]["cut"]
        strong = set(ws.strong_cuts(prob, cut).tolist())
        for L in CASES[name].longs:
            after = int(np.searchsorted(prob.in_start, prob.in_end[L.pos], "right"))
            if L.pos in strong and after in strong and after - L.pos >= ws.UNIT_MIN and not L.probe:
                hit.setdefault("strong cut before and after a long in-span", set()).add(name)
    prob = ws.strong_cut_case()
    cut = strong_cut_run()["sc"]["cut"]
    if ws.STRONG_Y not in ws.strong_cuts(prob, cut) and ws.STRONG_Y in ws.strong_cuts(prob, cut, wide_extent=False):
        hit.setdefault("cut kept from being strong by a wide in-span's extent alone", set()).add("strong-cut")
    print()
    for e in EDGES:
        print(f"{e:<56} {sorted(hit.get(e, ()))}")
    assert [e for e in EDGES if not hit.get(e)] == []


@pytest.mark.parametrize("name", SOLVED)
def test_generated_service(name):
    """Valid, in the two-pass regime, and wide where it should be: the oracle's scoring pass finishes and
    every long in-span has a feasible candidate past the narrow maps or shares a tile with one that does."""
    r = oracle_run(name)
    prob = r["prob"]
    assert prob.in_accelerated_regime()
    assert ws.wide_tiles(prob)
    ed = ws.edges(prob)
    for L in CASES[name].longs:
        assert L.pos // ws.SCORE_TILE in set(ws.wide_tiles(prob))
    # the host-side offsets agree with the oracle's feasible-tuple counts: an in-span with none has none
    assert np.array_equal(ed["off"].max(1) < 0, r["sc"]["n_feasible"] == 0)


def _bits_equal(a, b):
    return np.asarray(a, np.float64).tobytes() == np.asarray(b, np.float64).tobytes()


def assert_score_equal(got, ref, what):
    for k in ("cut", "n_feasible", "topk_cnt", "topk_idx"):
        assert np.array_equal(got[k], ref[k]), f"{what}: {k}"
    assert _bits_equal(got["topk_score"], ref["topk_score"]), f"{what}: topk_score"


def assert_stitch_equal(got, ref, what):
    for k in ("assign", "mis_rank", "n_cand", "topk_cnt", "topk_idx"):
        assert np.array_equal(got[k], ref[k]), f"{what}: {k}"
    assert _bits_equal(got["topk_score"], ref["topk_score"]), f"{what}: topk_score"
    assert np.array_equal(got["counters"][:, :2], ref["counters"][:, :2]), f"{what}: counters"


@pytest.mark.parametrize("backend", list(BACKENDS))
@pytest.mark.parametrize("name", SOLVED)
def test_stepped_device_code_equals_oracle(name, backend):
    r = oracle_run(name)
    eb = BACKENDS[backend](r["hb"])
    assert_score_equal(eb.score(gauss=r["gauss"]), r["sc"], "pass-0 score")
    assert eb.overflow == [64]               # the narrow maps overflowed: the wide maps re-ran the service
    assert_stitch_equal(eb.stitch(r["sc"]["cut"], gauss=r["gauss"]), r["st"], "pass-0 stitch")
    assert_score_equal(eb.score(mix=r["mix"]), r["sc1"], "pass-1 score")
    assert_stitch_equal(eb.stitch(r["sc"]["cut"], mix=r["mix"]), r["st1"], "pass-1 stitch")


def test_range_limit_at_offset_2048():
    """The wide maps hold feasible offsets 0 .. 2047 from lower_bound(start): offset 2047 scores, 2048 is
    TW_ERR_RANGE_LIMIT (as the redo kernel reports it), not a silently truncated map."""
    ok = EmulBatch(build_batch([problem("e1-off2047")]))
    ok.score(gauss=oracle_run("e1-off2047")["gauss"])
    assert ok.overflow == [64]
    hb = build_batch([problem("e1-off2048")])
    g = tw_oracle.OracleBatch(hb).params_pass0()
    with pytest.raises(_abi.TwError) as ei:
        EmulBatch(hb).score(gauss=g)
    assert ei.value.code == _abi.TW_ERR_RANGE_LIMIT


@lru_cache(maxsize=None)
def strong_cut_run():
    """The oracle's passes on tests/wide_synth.strong_cut_case()."""
    hb = build_batch([ws.strong_cut_case()])
    ob = tw_oracle.OracleBatch(hb)
    g = ob.params_pass0()
    sc = ob.score(gauss=g)
    st = ob.stitch(sc["cut"], gauss=g)
    d, c = ob.delays(st["assign"])
    mix, _, _ = tw_oracle.gmm_refit(hb.term_sample_off, d, c, seed_select=10)
    return dict(hb=hb, gauss=g, sc=sc, st=st, mix=mix, sc1=ob.score(mix=mix), st1=ob.stitch(sc["cut"], mix=mix))


@pytest.mark.parametrize("backend", list(BACKENDS))
def test_strong_cut_next_to_wide_in_span(backend):
    """The case is what it claims: cut[Y] = 1 is strong only without the wide in-span's extent, W takes c in
    pass 0 and q, whose only tuple uses c, stays unassigned; the stepped device code equals the oracle."""
    r = strong_cut_run()
    prob, n = ws.strong_cut_case(), int(r["hb"].prob_in_off[-1])
    cut, a = r["sc"]["cut"], r["st"]["assign"].reshape(prob.E, n)
    assert cut[ws.STRONG_Y] == 1 and ws.STRONG_Y >= ws.UNIT_MIN
    assert ws.STRONG_Y not in ws.strong_cuts(prob, cut)
    assert ws.STRONG_Y in ws.strong_cuts(prob, cut, wide_extent=False)
    assert (a[:, 0] >= 0).all() and r["sc"]["n_feasible"][ws.STRONG_Q] == 1
    assert (a[:, ws.STRONG_Q] == -1).all() and r["st"]["n_cand"][ws.STRONG_Q] == 0
    eb = BACKENDS[backend](r["hb"])
    assert_score_equal(eb.score(gauss=r["gauss"]), r["sc"], "pass-0 score")
    assert eb.overflow == [64]
    assert_stitch_equal(eb.stitch(r["sc"]["cut"], gauss=r["gauss"]), r["st"], "pass-0 stitch")
    assert_score_equal(eb.score(mix=r["mix"]), r["sc1"], "pass-1 score")
    assert_stitch_equal(eb.stitch(r["sc"]["cut"], mix=r["mix"]), r["st1"], "pass-1 stitch")
