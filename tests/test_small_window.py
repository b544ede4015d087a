"""The stitch kernel solves windows of <= 6 in-spans with a warp-parallel exhaustive search
(tw_stitch.cu: stitch_small_window) instead of the sequential branch and bound.  Its rule —
largest total, then the first leaf in depth-first order — must pick exactly what mwis_solve picks,
ties included.  Both are stepped on the CPU here (tests/emul): mwis_solve is the device function
itself, and so are the exhaustive search's leaves, each lane's running best and the butterfly merge of
the 32 lanes (tw_core.cuh); only the conflict masks the kernel takes from __match_any_sync are written
out for the CPU."""
import ctypes as C

import numpy as np
import pytest

import emul_backend


def _run(nw, E, cnt, score, idx):
    lib = emul_backend.lib()
    lib.twe_mwis_window.restype = C.c_longlong
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    cnt = np.ascontiguousarray(cnt, np.int32)
    score = np.ascontiguousarray(score, np.float64)
    idx = np.ascontiguousarray(idx, np.int32)
    a = np.full(nw, -9, np.int32)
    b = np.full(nw, -9, np.int32)
    nodes = lib.twe_mwis_window(nw, E, p(cnt), p(score), p(idx), p(a), C.c_longlong(10**7))
    assert nodes >= 0
    handled = lib.twe_small_window(nw, E, p(cnt), p(score), p(idx), p(b), 4096)
    return a, b, handled


@pytest.mark.parametrize("seed", range(300))
def test_exhaustive_search_equals_branch_and_bound(seed):
    _check(np.random.default_rng(seed), 1, 4, seed)


@pytest.mark.parametrize("seed", range(300, 900))
def test_exhaustive_search_equals_branch_and_bound_five_to_eight_callees(seed):
    """Tuples of 5..8 spans: the per-position conflict test runs over every callee, not the first four."""
    _check(np.random.default_rng(seed), 5, 8, seed)


def _check(rng, e_min, e_max, seed):
    nw = int(rng.integers(2, 7))
    E = int(rng.integers(e_min, e_max + 1))
    n_spans = int(rng.integers(2, 9))                      # few distinct spans: many conflicts
    cnt = rng.integers(0, 6, nw)
    score = np.full((nw, 5), np.nan)
    idx = np.full((nw, 5, E), -1, np.int32)
    levels = rng.choice([-3.0, -7.5, -12.25, -40.0, -20000.0], size=(nw, 5)) if seed % 3 == 0 else \
        -rng.exponential(25.0, size=(nw, 5))              # every third case: exact ties between totals
    for k in range(nw):
        score[k, :cnt[k]] = -np.sort(-levels[k, :cnt[k]])  # descending, like a top-K list
        idx[k, :cnt[k]] = rng.integers(0, n_spans, size=(cnt[k], E))
    a, b, handled = _run(nw, E, cnt, score, idx)
    if not handled:                                         # the kernel falls back to mwis_solve itself:
        assert E == 1 or np.prod(cnt + 1) > 4096            # Hungarian case, or too many leaves
        return
    assert np.array_equal(a, b), (cnt, score, idx)
