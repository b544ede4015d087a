"""tw_gmm_refit against the oracle's restated scikit-learn refit (oracle/tw_oracle_gmm.c) on the crafted delay
samples of tests/gmm_cases.py, at the random-stream positions the engine computes itself.

A case is compared only where gmm_cases.admit admits it: the oracle's fit agrees with its long double twin on
every decision and to 1e-11 on every BIC and parameter, no Lloyd label sits within rounding of a tie, and the
runner-up 'diag' BIC trails the selected one by at least 1e-7 |BIC|.  On those terms the selected K and rec[0] are exact,
pc and mu pc agree to 1e-9 relative, log pc and log w to 1e-9 absolute, and the degenerate record of a term
without a fit is bit-exact."""
import numpy as np
import pytest

import gmm_cases
from traceweaver_b200 import _abi, refit

pytestmark = pytest.mark.gpu

STREAM_LEN = 16384          # model-selection draws the engine generates (tw_api.cu kStreamLen)
RTOL, ATOL = 1e-9, 1e-9


@pytest.fixture(scope="module")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test needs a CUDA device")
    from traceweaver_b200.engine import Engine
    eng = Engine(0)
    yield eng
    eng.close()


def _batch(shape, n_terms, slot):
    """A bound batch of at least n_terms terms of `slot` samples each."""
    from traceweaver_b200 import synth
    from traceweaver_b200.batch import build_batch_from_blocks
    one = build_batch_from_blocks([synth.make_block(shape, 1, n_in=slot, seed=3)])
    per = int(one.ep_term_off[-1])
    return build_batch_from_blocks([synth.make_block(shape, -(-n_terms // per), n_in=slot, seed=3)])


def _fill(hb, samples):
    """delays / counts over the batch's term slots; terms past the cases hold no samples."""
    off = hb.term_sample_off
    nt = int(hb.ep_term_off[-1])
    assert len(samples) <= nt
    delays = np.zeros(int(off[-1]))
    counts = np.zeros(nt, np.int32)
    for t, x in enumerate(samples):
        assert len(x) <= off[t + 1] - off[t]
        delays[off[t]:off[t] + len(x)] = x
        counts[t] = len(x)
    return delays, counts


def _terms_of(hb, p):
    return int(hb.ep_term_off[hb.prob_ep_off[p]]), int(hb.ep_term_off[hb.prob_ep_off[p + 1]])


def _skips(hb, order, base, max_n):
    """Where each term's model-selection fits start: the problems' terms in `order`, from base[p] on."""
    skip = np.zeros(len(max_n), np.int64)
    for p in range(hb.n_problems):
        t0, t1 = _terms_of(hb, p)
        pos = int(base[p])
        for t in order[t0:t1]:
            skip[t] = pos
            pos += refit.draws_for(int(max_n[t]))
    return skip


def _refit(eng, hb, delays, counts, order=None, base=None):
    import torch
    eng.bind(hb)
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)
    prm, nsel = eng.gmm_refit(dev(delays), dev(counts), seed_select=10, prob_base_skip=dev(base),
                              term_order=dev(order), want_selected=True)
    eng.status()
    return prm.table.cpu().numpy(), nsel.cpu().numpy()


def _compare(names, got, gsel, want, wsel, ok):
    """Asserts the device records of the admitted terms; returns the largest differences seen."""
    worst = dict(pc=0.0, mupc=0.0, logpc=0.0, logw=0.0)
    for t, name in enumerate(names):
        if not ok[t]:
            continue
        assert gsel[t] == wsel[t], (name, gsel[t], wsel[t])
        assert got[t, 0] == want[t, 0], name
        k = int(want[t, 0])
        if k == 0:
            assert np.array_equal(got[t].view(np.uint64), want[t].view(np.uint64)), (name, got[t, :4], want[t, :4])
            continue
        for key, lo, rel in (("pc", 1, True), ("mupc", 6, True), ("logpc", 11, False), ("logw", 16, False)):
            g, w = got[t, lo:lo + k], want[t, lo:lo + k]
            d = np.abs(g - w) / (np.maximum(np.abs(w), np.finfo(float).tiny) if rel else 1.0)   # 0 only as 0
            worst[key] = max(worst[key], float(d.max()))
            assert d.max() <= (RTOL if rel else ATOL), (name, key, g, w)
    return worst


def _oracle(hb, delays, counts, skip):
    ok, reason, mix, nsel, _, _ = gmm_cases.admit(hb.term_sample_off, delays, counts, 10, skip.astype(np.uint32))
    return mix, nsel, ok, reason


def test_small_counts(engine):
    """Every case of up to 4224 samples as one term of one bound batch: a permuted term order, a nonzero
    base position per problem, and one term whose first 2-component draw lands in the replay band."""
    cs = gmm_cases.cases()
    n_rp, pos_rp = gmm_cases.replay_position(range(2, 4225))
    cs.append((f"replay-n{n_rp}", gmm_cases.sample("one_cluster", n_rp, 1)))
    hb = _batch("hotel_frontend", len(cs), max(gmm_cases.N_SMALL))
    names = [c[0] for c in cs] + ["empty"] * (int(hb.ep_term_off[-1]) - len(cs))
    delays, counts = _fill(hb, [c[1] for c in cs])
    cap = refit.unique_cap(delays, hb.term_sample_off, counts)
    rng = np.random.default_rng(5)
    order = np.arange(len(counts), dtype=np.int32)
    base = ((np.arange(hb.n_problems) * 997 + 11) % (STREAM_LEN // 2)).astype(np.uint32)
    for p in range(hb.n_problems):
        t0, t1 = _terms_of(hb, p)
        order[t0:t1] = t0 + rng.permutation(t1 - t0)
    # the replay term (last case) first in its problem's order, its K = 2 fit starting at pos_rp
    t_rp = len(cs) - 1
    p_rp = int(np.searchsorted(hb.ep_term_off[hb.prob_ep_off], t_rp, side="right")) - 1
    t0, t1 = _terms_of(hb, p_rp)
    rest = [t for t in order[t0:t1] if t != t_rp]
    order[t0:t1] = [t_rp] + rest
    assert cap[t_rp] >= 2
    base[p_rp] = pos_rp - refit.draws_for(1)
    skip = _skips(hb, order, base, cap)
    assert skip[t_rp] + refit.draws_for(1) == pos_rp

    got, gsel = _refit(engine, hb, delays, counts, order, base)
    # the stream bookkeeping: per-problem draws of a model-selection pass
    import torch
    drawn = engine.gmm_stream_draws(torch.from_numpy(delays).to(engine.device),
                                    torch.from_numpy(counts).to(engine.device)).cpu().numpy()
    for p in range(hb.n_problems):
        t0, t1 = _terms_of(hb, p)
        assert drawn[p] == sum(refit.draws_for(int(m)) for m in cap[t0:t1]), p
    want, wsel, ok, reason = _oracle(hb, delays, counts, skip)
    assert ok[t_rp]
    worst = _compare(names, got, gsel, want, wsel, ok)
    rejected = {}
    for t in range(len(cs)):
        if not ok[t]:
            rejected[reason[t]] = rejected.get(reason[t], 0) + 1
    print(f"\nsmall counts: {len(cs)} cases, {len(cs) - sum(rejected.values())} admitted, rejected {rejected}; "
          f"largest differences {worst}")


def test_stream_end(engine):
    """A model-selection pass whose last fit ends exactly at draw 16384 runs; one draw later is
    TW_ERR_RANGE_LIMIT."""
    cs = [(f"{k}-n{n}", gmm_cases.sample(k, n, 2)) for n in (64, 1025) for k in ("three_equal", "negative")]
    hb = _batch("hotel_search", len(cs), 1025)
    names = [c[0] for c in cs] + ["empty"] * (int(hb.ep_term_off[-1]) - len(cs))
    delays, counts = _fill(hb, [c[1] for c in cs])
    cap = refit.unique_cap(delays, hb.term_sample_off, counts)
    order = np.arange(len(counts), dtype=np.int32)
    base = np.zeros(hb.n_problems, np.uint32)
    for p in range(hb.n_problems):
        t0, t1 = _terms_of(hb, p)
        base[p] = STREAM_LEN - sum(refit.draws_for(int(m)) for m in cap[t0:t1])
    got, gsel = _refit(engine, hb, delays, counts, order, base)
    want, wsel, ok, _ = _oracle(hb, delays, counts, _skips(hb, order, base, cap))
    worst = _compare(names, got, gsel, want, wsel, ok)
    print(f"\nstream end: {int(ok[:len(cs)].sum())} of {len(cs)} admitted; largest differences {worst}")
    base += 1
    with pytest.raises(_abi.TwError) as ex:
        _refit(engine, hb, delays, counts, order, base)
    assert ex.value.code == _abi.TW_ERR_RANGE_LIMIT


@pytest.mark.parametrize("ns", [gmm_cases.N_LARGE, [485371]], ids=["16385-30000", "485371"])
def test_large_counts(engine, ns):
    """Past LogSum's flush and Lloyd's shared-memory labels; at 485371 samples the final fit's first draw of
    RandomState(100) lies where floor(u n) is one off NumPy's first centre."""
    kinds = ("one_cluster", "three_equal", "two_skewed", "int_us") if len(ns) > 1 else ("three_equal",)
    cs = [(f"{k}-n{n}", gmm_cases.sample(k, n, 4)) for n in ns for k in kinds]
    hb = _batch("single", len(cs), max(ns))
    names = [c[0] for c in cs] + ["empty"] * (int(hb.ep_term_off[-1]) - len(cs))
    delays, counts = _fill(hb, [c[1] for c in cs])
    cap = refit.unique_cap(delays, hb.term_sample_off, counts)
    order = np.arange(len(counts), dtype=np.int32)
    got, gsel = _refit(engine, hb, delays, counts)
    want, wsel, ok, _ = _oracle(hb, delays, counts, _skips(hb, order, np.zeros(hb.n_problems), cap))
    worst = _compare(names, got, gsel, want, wsel, ok)
    print(f"\nlarge counts {ns}: {int(ok[:len(cs)].sum())} of {len(cs)} admitted; largest differences {worst}")
    if ns == [485371]:
        # RandomState(100)'s first draw puts u n 2.0e-6 above 263753: floor(u n) takes sample 263753,
        # NumPy's cumulative sum sample 263752.  A build with the fixed 1e-6 replay band started the final fit
        # from the other centre and returned the same components in another order.
        assert ok[0] and wsel[0] >= 2
