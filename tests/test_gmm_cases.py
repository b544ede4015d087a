"""The crafted delay samples of tests/gmm_cases.py (compared with the device in test_gpu_gmm_refit.py): they are
deterministic, they reach the shapes they are named for, and the oracle fits every one of them."""
import os

import numpy as np

import gmm_cases
from oracle import tw_oracle
from traceweaver_b200 import refit


def _run(cs):
    counts = np.array([len(x) for _, x in cs], np.int32)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    delays = np.concatenate([x for _, x in cs])
    return delays, off, counts


def test_cases_are_deterministic():
    a, b = gmm_cases.cases(), gmm_cases.cases()
    assert [n for n, _ in a] == [n for n, _ in b]
    assert all(np.array_equal(x.view(np.uint64), y.view(np.uint64)) for (_, x), (_, y) in zip(a, b))


def test_cases_reach_their_shapes():
    # k_gmm_prep: each lane's local five-value set fills with values the other lanes' sets do not hold first
    x = gmm_cases.sample("lane_sets", 4224, 0)
    lane_sets = [tuple(dict.fromkeys(x[l::32]))[:5] for l in range(32)]
    assert len(set(lane_sets)) == 32
    assert len(np.unique(x)) == 37
    z = gmm_cases.sample("signed_zero", 64, 0)
    assert np.signbit(z[z == 0.0]).any() and not np.signbit(z[z == 0.0]).all()
    assert len(np.unique(z)) == 3
    assert np.all(gmm_cases.sample("dyadic", 1024, 0) * 64.0 % 1.0 == 0.0)
    assert np.all(gmm_cases.sample("int_us", 1024, 0) % 1.0 == 0.0)
    assert (gmm_cases.sample("negative", 1024, 0) < 0).any()
    lone = gmm_cases.sample("lone_sample", 33, 0)
    assert np.count_nonzero(lone > 30000) == 1


def test_oracle_fits_every_case():
    cs = gmm_cases.cases()
    delays, off, counts = _run(cs)
    cap = refit.unique_cap(delays, off, counts)
    mix, nsel, max_n = tw_oracle.gmm_refit(off, delays, counts, seed_select=10)
    _, _, _, bic, _ = tw_oracle.gmm_refit(off, delays, counts, seed_select=10, want_record=True)
    assert np.array_equal(max_n, cap)
    for t, (name, x) in enumerate(cs):
        n = len(x)
        if n < 2:                                  # no fit is tried: the degenerate record
            assert nsel[t] == 0 and mix[t, 2] == 0.001, name
            continue
        assert 1 <= nsel[t] <= min(cap[t], n), name
        assert np.isfinite(bic[t, nsel[t] - 1]) and bic[t, nsel[t] - 1] == np.min(bic[t]), name
        assert np.all(np.isinf(bic[t, cap[t]:])), name


# branches of the refit no generated case reaches: scikit-learn's ValueError needs a covariance <= 0 after
# reg_covar, k-means' empty-cluster relocation never occurred in 20 000 random 1-D k-means++ runs, and EM
# converges well within 100 iterations on every case
UNREACHED = {"ValueError", "relocation", "EM not converged"}


def test_admitted_cases_cover_the_branches():
    """Each branch of the fit occurs in at least one admitted case; the replay of the first centre on a term
    placed at the draw where it runs."""
    cs = gmm_cases.cases()
    n_rp, pos_rp = gmm_cases.replay_position(range(2, 4225))
    cs.append(("replay", gmm_cases.sample("one_cluster", n_rp, 1)))
    delays, off, counts = _run(cs)
    skip = np.zeros(len(cs), np.uint32)
    skip[-1] = pos_rp - refit.draws_for(1)           # its 2-component fit draws the first centre at pos_rp
    ok, reason, _, nsel, _, rec = gmm_cases.admit(off, delays, counts, 10, skip)
    F = {f: i for i, f in enumerate(tw_oracle.GMM_REC_FIELDS)}
    a = rec[ok]
    fitted = a[:, :, F["status"]] == 1
    seen = {"too few samples": (a[:, :, F["status"]] == -1).any(),
            "ValueError": (a[:, :, F["status"]] == -2).any(),
            "fitted": fitted.any(),
            "Lloyd strict stop": (fitted & (a[:, :, F["lloyd_iter"]] > 0) & (a[:, :, F["lloyd_strict"]] == 1)).any(),
            "Lloyd tol stop": (fitted & (a[:, :, F["lloyd_iter"]] > 0) & (a[:, :, F["lloyd_strict"]] == 0)).any(),
            "relocation": (a[:, :, F["relocations"]] > 0).any(),
            "EM converged": (fitted & (a[:, :, F["em_converged"]] == 1)).any(),
            "EM not converged": (fitted & (a[:, :, F["em_converged"]] == 0)).any(),
            "replay": (a[:, :, F["replay"]] == 1).any(),
            "no fit (degenerate record)": (nsel[ok] == 0).any()}
    reached = {b for b, v in seen.items() if v}
    assert ok[-1], reason[-1]
    assert reached == set(seen) - UNREACHED, (reached, UNREACHED)
    rejected = {}
    for r in reason:
        if r:
            rejected[r] = rejected.get(r, 0) + 1
    print(f"\n{len(cs)} cases, {int(ok.sum())} admitted, rejected {rejected}; unreached branches {sorted(UNREACHED)}")


def test_admission_rejects_the_ill_conditioned_golden_terms():
    """The hand lists of ill-conditioned golden terms (test_oracle_gmm.py, test_gpu_pipeline.py) are all
    rejected by the long double twin; prints how many golden terms it admits."""
    from test_gpu_pipeline import ILL_CONDITIONED as PIPE
    from test_oracle_gmm import ILL_CONDITIONED as ORACLE, _setup
    from golden_util import golden_files
    hand = {(k, t) for d in (ORACLE, PIPE) for k, ts in d.items() for t in ts}
    assert len(hand) == 4
    admitted = total = 0
    seen = set()
    for path in golden_files():
        name = os.path.basename(path)[:-4]
        g, _, hb, d, c, skips = _setup(path)
        ok, reason, *_ = gmm_cases.admit(hb.term_sample_off, d, c, g.meta["global_seed"], skips)
        for t in range(len(c)):
            if (name, t) in hand:
                assert not ok[t], (name, t)
                seen.add((name, t))
                print(f"\n{name} term {t}: {reason[t]}")
        admitted += int(ok.sum())
        total += len(c)
    assert seen == hand
    print(f"\ngolden terms admitted: {admitted} of {total}")
