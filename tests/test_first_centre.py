"""The refit's first k-means++ centre (first_centre, tw_core.cuh, on the CPU through tests/emul) against
NumPy's RandomState.choice(n, p=np.full(n, 1/n)), which scikit-learn's _kmeans_plusplus calls.

NumPy's cumulative sum of 1/n drifts from (i + 1)/n by up to about n^2 2^-53 in units of u n, so floor(u n)
is NumPy's index only away from that band.  The draws here sit at fractions and multiples of n^2 2^-53
around chosen integers, including those where the drift is largest; floor(u n) with a fixed 1e-6 replay
band gets some of them wrong from a few 10^4 samples on."""
import numpy as np
import pytest

import emul_backend

# every n the first centre has been seen to go wrong at, the warp and Lloyd boundaries of tw_gmm.cu, and
# a geometric ladder up to 2^24
NAMED = [30000, 300000, 485371, 500000, 888908, 943464, 1000000, 3000000]
NS = sorted(set(range(1, 66)) | {127, 128, 129, 1023, 1024, 1025, 4095, 4096, 4097, 16385, 65536, 131071}
            | {int(v) for v in np.geomspace(100, 2 ** 24, 24)} | set(NAMED) | {2 ** 24})


def _cdf(n):
    """choice()'s cdf for p = np.full(n, 1/n) (numpy/random/mtrand.pyx: cumsum, then divide by the last)."""
    cdf = np.cumsum(np.full(n, 1.0 / n))
    cdf /= cdf[-1]
    return cdf


def _numpy_index(cdf, u):
    return np.searchsorted(cdf, u, side="right")


def _old_rule(cdf, u, n):
    """The rule of earlier builds: floor(u n), replayed only within 1e-6 of an integer."""
    un = u * n
    return np.where(np.abs(un - np.rint(un)) < 1e-6, _numpy_index(cdf, u), np.minimum(np.floor(un), n - 1))


def _draws(n, cdf):
    """u at ±(0, 0.001, 0.01, 0.1, 1, 10, 100, 1000) n^2 2^-53 around a few integers and around the
    integers of largest drift, and halfway between those integers and n cdf_i (the measured drift is about
    a tenth of n^2 2^-53, so the band floor(u n) misses lies below the unit multiple)."""
    drift = cdf * n - np.arange(1, n + 1)
    worst = np.argsort(np.abs(drift))[-3:]
    js = {1, n // 3, n // 2, n - 1} | {int(i) + 1 for i in worst}   # cdf_i crosses u near u n = i + 1
    step = float(n) * n * 2.0 ** -53
    us = [(j + s * m * step) / n for j in js for m in (0, 1e-3, 1e-2, 0.1, 1, 10, 100, 1000) for s in (1, -1)]
    us += [(i + 1 + 0.5 * drift[i]) / n for i in worst]
    return np.unique(np.array([u for u in us if 0.0 <= u < 1.0]))


def test_choice_is_the_cumulative_sum():
    """The restatement above is RandomState.choice itself: at the first draws of the seeds the refit uses."""
    for n in (1, 2, 5, 1000, 1025, 30000, 485371, 1000000):
        p = np.full(n, 1.0 / n)
        cdf = _cdf(n)
        for seed in (10, 100, 7):
            u = np.random.RandomState(seed).random_sample(4)
            r = np.random.RandomState(seed)
            got = [r.choice(n, p=p) for _ in range(4)]
            assert got == _numpy_index(cdf, u).tolist(), (n, seed)


def test_first_centre_matches_numpy():
    old_wrong = 0
    for n in NS:
        cdf = _cdf(n)
        u = _draws(n, cdf)
        want = _numpy_index(cdf, u)
        got = emul_backend.first_centre(u, n)
        bad = np.nonzero(got != want)[0]
        assert len(bad) == 0, (n, u[bad[:5]], got[bad[:5]], want[bad[:5]])
        old_wrong += int(np.count_nonzero(_old_rule(cdf, u, n) != want))
    # the cases reach the band the fixed 1e-6 replay missed
    assert old_wrong > 0
    print(f"first_centre == RandomState.choice at {len(NS)} sample counts; the old rule misses {old_wrong} draws")


@pytest.mark.parametrize("n,want", [(485371, 263752), (888908, 483037), (943464, None)])
def test_final_fit_first_draw(n, want):
    """The final 'full' fit draws from RandomState(100): its first centre at the counts where floor(u n)
    is one off NumPy's index."""
    p = np.full(n, 1.0 / n)
    ref = int(np.random.RandomState(100).choice(n, p=p))
    if want is not None:
        assert ref == want
    u0 = np.random.RandomState(100).random_sample()
    assert int(np.floor(u0 * n)) != ref                   # the draw sits in the drift band
    assert int(emul_backend.first_centre(u0, n)[0]) == ref


def test_model_selection_stream():
    """At n = 10^6 some of the first 2·10^6 draws of seed 10 fall in the drift band; at each of them the first
    centre is choice()'s index, taken from a RandomState advanced to that draw."""
    n = 1000000
    cdf = _cdf(n)
    u = np.random.RandomState(10).random_sample(2000000)
    want = _numpy_index(cdf, u)
    pos = np.nonzero(_old_rule(cdf, u, n) != want)[0]
    assert len(pos) > 0 and pos[0] == 19345, pos[:6]
    got = emul_backend.first_centre(u[pos], n)
    assert np.array_equal(got, want[pos])
    p = np.full(n, 1.0 / n)
    for q in pos[:2]:
        r = np.random.RandomState(10)
        r.random_sample(int(q))
        assert int(r.choice(n, p=p)) == int(want[q])
