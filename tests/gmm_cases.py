"""Deterministic delay samples for the refit's device-vs-oracle test (tests/test_gpu_gmm_refit.py).  Seeds
only, no stored data.

Sample counts sit at the kernels' own boundaries (tw_gmm.cu): a fit needs n >= 2 and n >= K; sweep2 takes
each lane's samples in pairs, 32 lanes to a warp; Lloyd keeps its labels in shared memory up to
kLloydLabelN = 1024 samples and recomputes them above; LogSum flushes its product after 128 samples per
lane (n > 4096).  The value shapes are well-separated continuous clusters (one to six, equal and skewed
weights, one lone sample), integer microseconds, multiples of 1000 (millisecond clocks), multiples of 2^-6,
negative delays, values near 1e7 with a spread of about 10, one to six distinct values, for k_gmm_prep lanes
whose local five-value sets fill with different values (an evenly spaced grid) and -0.0 mixed with 0.0.

`admit` decides which terms a device-vs-oracle comparison may check: those whose oracle fit does not depend
on summation order."""
import numpy as np

from oracle import tw_oracle

N_SMALL = [0, 1, 2, 3, 4, 5, 6, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1023, 1024, 1025, 1087, 4095, 4096, 4097,
           4224]
N_LARGE = [16385, 30000]
KINDS = ("one_cluster", "three_equal", "two_skewed", "four_clusters", "six_clusters", "lone_sample", "int_us",
         "ms_clock", "dyadic", "negative", "near_1e7", "distinct1", "distinct2", "distinct3", "distinct4",
         "distinct5", "distinct6", "lane_sets", "signed_zero")
# admission (admit): the long double build agrees to this relative difference, and the runner-up BIC trails
# the selected one by at least GAP |BIC|
TWIN_RTOL = 1e-11
GAP = 1e-7


def _clusters(rng, n, centres, sds, weights):
    lab = rng.choice(len(centres), size=n, p=np.asarray(weights) / np.sum(weights))
    return np.asarray(centres, float)[lab] + rng.normal(size=n) * np.asarray(sds, float)[lab]


def _distinct(rng, n, values):
    v = np.asarray(values, float)
    return v[np.arange(n) % len(v)][rng.permutation(n)] if n else np.zeros(0)


def sample(kind, n, seed):
    """n delays (float64) of one value shape, from a seed."""
    rng = np.random.default_rng([seed, n, KINDS.index(kind)])
    if kind == "one_cluster":
        return rng.normal(5000.0, 300.0, n)
    if kind == "three_equal":
        return _clusters(rng, n, [1000, 5000, 20000], [40, 150, 600], [1, 1, 1])
    if kind == "two_skewed":
        return _clusters(rng, n, [2000, 12000], [100, 500], [0.9, 0.1])
    if kind == "four_clusters":
        return _clusters(rng, n, [500, 2000, 8000, 30000], [20, 80, 300, 1000], [4, 1, 2, 1])
    if kind == "six_clusters":
        return _clusters(rng, n, [300, 1000, 3000, 9000, 27000, 81000], [10, 30, 100, 300, 900, 2700], [1] * 6)
    if kind == "lone_sample":               # one sample far from the rest: a one-sample component
        x = rng.normal(3000.0, 200.0, n)
        if n:
            x[rng.integers(n)] = 60000.0
        return x
    if kind == "int_us":
        return np.rint(rng.lognormal(np.log(3000.0), 0.5, n))
    if kind == "ms_clock":                  # millisecond clocks: few distinct multiples of 1000
        return np.rint(rng.lognormal(np.log(3000.0), 0.5, n) / 1000.0) * 1000.0
    if kind == "near_1e7":                  # 'diag' covariance avg(x^2) - mean^2 cancels 12 digits
        return 1e7 + rng.normal(0.0, 10.0, n)
    if kind == "dyadic":                    # multiples of 2^-6
        return np.round(_clusters(rng, n, [300, 900], [20, 40], [1, 2]) * 64.0) / 64.0
    if kind == "negative":
        return _clusters(rng, n, [-2000, 3000], [100, 200], [1, 1])
    if kind.startswith("distinct"):
        return _distinct(rng, n, 1000.0 * 3.0 ** np.arange(int(kind[len("distinct"):])))
    if kind == "lane_sets":                 # lane l sees values l, l + 32, ... (mod 37): every lane's set fills
        return (np.arange(n) % 37) * 250.0 + 1000.0
    if kind == "signed_zero":               # np.unique and the device both take -0.0 == 0.0
        return _distinct(rng, n, [-0.0, 0.0, 4000.0, 0.0, 20000.0, -0.0])
    raise ValueError(kind)


def replay_position(ns, stream_len=16384):
    """(n, draw position) of the first draw in the first half of the seed-10 model-selection stream at which
    some n of `ns` puts u n within 1e-6 of an integer, the band where the seeding replays NumPy's cumulative
    sum (first_centre, tw_core.cuh)."""
    u = np.random.RandomState(10).random_sample(stream_len)[:stream_len // 2]
    for n in ns:
        un = u * n
        hit = np.nonzero(np.abs(un[1:] - np.rint(un[1:])) < 1e-6)[0] + 1
        if len(hit):
            return n, int(hit[0])
    raise ValueError("no draw in the replay band")


def cases(ns=N_SMALL, seed=0):
    """[(name, samples)] over ns x KINDS."""
    return [(f"{k}-n{n}", sample(k, n, seed)) for n in ns for k in KINDS]


def admit(term_sample_off, delays, counts, seed_select=10, rng_skip=None):
    """The oracle's refit of every term (two_gmm_refit_record) and which terms it admits: the double and the
    long double builds agree on every decision (selected K, #unique cap, every field of every fit's record),
    every per-K 'diag' BIC and every parameter of the final record agree to TWIN_RTOL, no Lloyd label is
    within rounding of a tie (the long double build sums the centres more exactly but measures distances the
    same way, so it cannot see a sample that sits exactly between two centres), and the runner-up BIC trails
    the selected one by at least GAP |BIC|.  Returns (ok, reason per term, mix, nsel, bic, rec)."""
    args = (term_sample_off, delays, counts, seed_select, rng_skip)
    mix, nsel, max_n, bic, rec = tw_oracle.gmm_refit(*args, want_record=True)
    mix2, nsel2, max_n2, bic2, rec2 = tw_oracle.gmm_refit(*args, want_record=True, twin=True)

    def close(a, b):
        with np.errstate(invalid="ignore"):
            return (a == b) | (np.abs(a - b) <= TWIN_RTOL * np.maximum(np.abs(a), np.abs(b)))

    reason = []
    for t in range(len(counts)):
        b = np.sort(bic[t][np.isfinite(bic[t])])
        if nsel[t] != nsel2[t] or max_n[t] != max_n2[t] or not np.array_equal(rec[t], rec2[t]):
            reason.append("decisions differ in long double")
        elif not close(bic[t], bic2[t]).all():
            reason.append("BIC differs in long double")
        elif not close(mix[t], mix2[t]).all():
            reason.append("parameters differ in long double")
        elif rec[t, :, tw_oracle.GMM_REC_FIELDS.index("lloyd_ties")].any():
            reason.append("Lloyd label within rounding of a tie")
        elif len(b) > 1 and b[1] - b[0] < GAP * abs(b[0]):
            reason.append("BIC gap")
        else:
            reason.append("")
    ok = np.array([r == "" for r in reason])
    return ok, reason, mix, nsel, bic, rec
