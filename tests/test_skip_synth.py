"""Skip regime on generated cache-mode services (tests/skip_synth.py), CPU only: the device code of
k_skip (tw_skip_core.cuh) stepped on the CPU and the host mirror's NumPy tally against the oracle
(oracle/tw_oracle_skip.py), over every synthetic shape, the eight-callee DAG, microsecond and
millisecond clocks, both budget signs, carried windows and samples, and the reference's error cases.
The emulator is fed the model the oracle's own pieces build (windows, skip counts, services_times), so
the cases where the reference raises are compared too."""
import numpy as np
import pytest

import skip_synth as ss
from oracle import tw_oracle_skip as osk
from traceweaver_b200 import _abi, skipmode

CASES = ss.matrix()
IDS = [name for name, _ in CASES]


@pytest.fixture(scope="module")
def oracle_runs():
    """name -> (service, oracle result or the ReferenceUndefined it raised, branch counts, model)."""
    runs = {}

    def get(name):
        if name not in runs:
            svc = dict(CASES)[name]()
            runs[name] = (svc,) + ss.run_oracle(svc)
        return runs[name]
    return get


def _emul(svc, md):
    import emul_backend
    return emul_backend.skip_solve(svc.in_start, svc.in_end, svc.out_start, svc.out_end, svc.preds, md["wins"],
                                   md["counts"], md["tab"], md["budgets"])


@pytest.mark.parametrize("name", IDS)
def test_device_code_stepped_on_cpu_equals_oracle(oracle_runs, name):
    svc, ref, _, md = oracle_runs(name)
    if isinstance(ref, osk.ReferenceUndefined):
        with pytest.raises(_abi.TwError) as ex:
            _emul(svc, md)
        assert ex.value.code == _abi.TW_ERR_REFERENCE_UNDEFINED, str(ref)
        return
    # the model the emulator is given is the oracle's own
    assert ref["time_windows"] == md["wins"] and ref["skip_budget"] == md["budgets"]
    assert ref["skip_count"] == md["counts"]
    assert np.array_equal(ref["pair_params"], md["tab"], equal_nan=True)
    ss.assert_equals_oracle(_emul(svc, md), ref)


@pytest.mark.parametrize("name", IDS)
def test_host_mirror_tally_equals_oracle(oracle_runs, name):
    """Time windows, budgets and water-filled skip counts of traceweaver_b200.skipmode (NumPy)."""
    svc, _, _, md = oracle_runs(name)
    st = skipmode.SkipState()
    st.time_windows = list(svc.wins_before)
    _, s_start, _ = skipmode.sort_partitions(svc.out_start, svc.out_end)
    wins, budgets, counts = skipmode.tally(svc.in_start, svc.in_end, s_start, st)
    assert wins == md["wins"] and budgets == md["budgets"]
    assert np.array_equal(counts, np.asarray(md["counts"]))


@pytest.mark.parametrize("n_cand", [96, 97])
def test_candidate_limit_stepped_on_cpu(n_cand):
    """kSkipCand = 96 candidates of one callee inside one in-span: 96 solve like the oracle, 97 are
    TW_ERR_RANGE_LIMIT (no partial answer comes back)."""
    svc = ss.cand_limit_service(n_cand)
    ref, _, md = ss.run_oracle(svc)
    assert not isinstance(ref, Exception)
    inside = [int(((o >= s) & (x <= e)).sum()) for s, e in zip(svc.in_start, svc.in_end)
              for o, x in zip(svc.out_start[:1], svc.out_end[:1])]
    assert max(inside) == n_cand
    if n_cand <= 96:
        ss.assert_equals_oracle(_emul(svc, md), ref)
    else:
        with pytest.raises(_abi.TwError) as ex:
            _emul(svc, md)
        assert ex.value.code == _abi.TW_ERR_RANGE_LIMIT


def branch_table(oracle_runs):
    """Cases reaching each branch the skip tests are meant to cover (oracle counts and input features)."""
    rows = {f"E={e}": 0 for e in (1, 2, 3, 4, 8)}
    rows.update({k: 0 for k in ("normalized=0", "mixed budget signs", "skip_pred_root", "skip_pred_ancestor",
                                "non_primary_edge", "err_ancestor_chain", "tie_real_real", "err_tie_skip_real",
                                "err_all_skip", "err_missing_key", "unsorted caller list", "equal starts in a list",
                                "in-span in a window with a shared start", "TW_ERR_REFERENCE_UNDEFINED")})
    for name in IDS:
        svc, ref, counts, md = oracle_runs(name)
        for k, v in list(counts.items()) + list(ss.input_features(svc, md).items()):
            if v and k in rows:
                rows[k] += 1
        rows["TW_ERR_REFERENCE_UNDEFINED"] += isinstance(ref, osk.ReferenceUndefined)
    return rows


def test_every_branch_is_reached(oracle_runs):
    """The generated matrix keeps reaching every branch (TW_ERR_RANGE_LIMIT: test_candidate_limit_*)."""
    rows = branch_table(oracle_runs)
    print("\n" + "\n".join(f"{k:45s} {v:4d}" for k, v in rows.items()))
    assert all(v > 0 for v in rows.values()), {k: v for k, v in rows.items() if v == 0}
