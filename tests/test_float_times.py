"""CPU side of the float64-timestamp path (time-compressed services, executor.py --compress_factor > 1):
the float64 build of the oracle, the fixed-point shift rule, and the precondition under which the
engine's results must coincide with the reference's on the fractional test inputs."""
import math

import numpy as np
import pytest

from float_times_util import FIXED_BITS, compress, reference_sums_exact, shift_rule, times
from golden_util import Golden, golden_files

FILES = golden_files()
IDS = [f.split("/")[-1][:-4] for f in FILES]
FACTORS = (3, 200, 15000)


def _float_copy(prob):
    from traceweaver_b200.batch import Problem
    f = lambda a: np.asarray(a, np.int64).astype(np.float64)
    return Problem(in_start=f(prob.in_start), in_end=f(prob.in_end), out_start=[f(a) for a in prob.out_start],
                   out_end=[f(a) for a in prob.out_end], preds=prob.preds, name=prob.name)


@pytest.mark.parametrize("path", FILES, ids=IDS)
def test_float_oracle_equals_int_oracle_on_integral_inputs(path):
    import oracle_f64
    from oracle import tw_oracle
    from traceweaver_b200.batch import build_batch
    prob = Golden(path).problem()
    hi, hf = build_batch([prob]), build_batch([_float_copy(prob)])
    assert hf.float_times and not hi.float_times
    oi, of = tw_oracle.OracleBatch(hi), oracle_f64.OracleBatch(hf)
    gi, gf = oi.params_pass0(), of.params_pass0()
    assert gi.tobytes() == gf.tobytes()
    si, sf = oi.score(gauss=gi), of.score(gauss=gf)
    for k in si:
        assert si[k].tobytes() == sf[k].tobytes(), k
    ri, rf = oi.stitch(si["cut"], gauss=gi), of.stitch(sf["cut"], gauss=gf)
    for k in ri:
        assert ri[k].tobytes() == rf[k].tobytes(), k
    di, df = oi.delays(ri["assign"]), of.delays(rf["assign"])
    assert di[0].tobytes() == df[0].tobytes() and di[1].tobytes() == df[1].tobytes()
    ai, af = tw_oracle.find_assignments(hi, 10), oracle_f64.find_assignments(hf, 10)
    for k in ai:
        assert ai[k].tobytes() == af[k].tobytes(), k


def test_shift_rule_on_crafted_values():
    assert shift_rule([0.0, 1.0, -5.0, 1655000000004518.0]) == 0             # integers
    assert shift_rule([1.5, 2.25]) == 2
    x = [float(v) / 3 for v in (1655000000004518, 1655000000009640)]         # x / 3: ~2^48.97, 52-bit mantissas
    assert shift_rule(x) == 52 - 48
    s = shift_rule([float(2 ** 40) - 0.5 ** 12, float(2 ** 40) + 0.5 ** 11])  # binade straddle: the finer side wins
    assert s == 12
    for bad in (math.nan, math.inf, -math.inf):
        assert shift_rule([1.0, bad]) is None
    assert shift_rule([2.0 ** FIXED_BITS]) is None                           # max|x| * 2^s >= 2^55
    assert shift_rule([2.0 ** FIXED_BITS - 8]) == 0
    assert shift_rule([2.0 ** 51 + 0.5]) == 1                                # X = 2^52 + 1 fits
    assert shift_rule([2.0 ** 51 + 0.5, 2.0 ** 54]) is None                  # the resolution of one, the size of the other


def test_fixed_point_is_exact_and_monotone():
    prob = compress(Golden(FILES[0]).problem(), 200)
    v = np.sort(np.concatenate(times(prob)))
    s = shift_rule(v)
    X = [math.ldexp(float(x), s) for x in v]
    assert all(float(int(x)) == x and abs(x) < 2.0 ** FIXED_BITS for x in X)
    assert all(a <= b for a, b in zip(X, X[1:]))
    a, b = float(v[-1]), float(v[0])
    assert math.ldexp(int(X[-1]) - int(X[0]), -s) == a - b                 # (X_a - X_b) 2^-s == x_a - x_b


@pytest.mark.parametrize("cf", FACTORS)
@pytest.mark.parametrize("path", FILES, ids=IDS)
def test_fractional_inputs_are_in_the_exact_regime(path, cf):
    """The fractional test inputs meet the condition under which the reference's own double arithmetic is
    exact, so engine == float oracle there is the statement that matters."""
    prob = compress(Golden(path).problem(), cf)
    assert shift_rule(np.concatenate(times(prob))) is not None
    assert reference_sums_exact(prob)
