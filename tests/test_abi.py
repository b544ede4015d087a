"""CPU-side checks of the C-ABI library: it loads, exports every symbol the header declares, and
validates descriptors on the host (no compute without a GPU)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from traceweaver_b200 import _abi, _lib
from traceweaver_b200.batch import Problem, build_batch, batch_struct

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from traceweaver_b200.csrc import build
    build.build()
    return _lib.load()


def test_every_declared_symbol_is_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "traceweaver_b200.h")).read()
    declared = set(re.findall(r"^\s*(?:int|int64_t|const char\*)\s+(tw_[a-z0-9_]+)\s*\(", hdr, re.M))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.SYMBOLS), (declared ^ set(_lib.SYMBOLS))
    for name in declared:
        assert hasattr(lib, name)
    assert lib.tw_abi_version() == _abi.TW_ABI_VERSION


def _toy(n=6, E=2):
    s = np.arange(n, dtype=np.int64) * 1000
    return Problem(in_start=s, in_end=s + 900, out_start=[s + 10 * (e + 1) for e in range(E)],
                   out_end=[s + 10 * (e + 1) + 5 for e in range(E)], preds=[[], [0]][:E], name="toy")


def test_struct_layout_matches_header(lib):
    # sizes follow from the header's field list: 4 int32 + 2 int64 + 11 pointers
    assert C.sizeof(_abi.TwBatch) == 16 + 16 + 11 * 8
    assert C.sizeof(_abi.TwParams) == 8 + 3 * 8
    assert C.sizeof(_abi.TwPassOut) == 7 * 8
    assert C.sizeof(_abi.TwScoreOut) == 9 * 8
    assert C.sizeof(_abi.TwSkipDesc) == 10 * 8
    assert C.sizeof(_abi.TwTraceKeys) == 4 * 8 + 8
    assert C.sizeof(_abi.TwSkipOut) == 7 * 8 + 4 * 8


def test_host_validation(lib):
    hb = build_batch([_toy()])
    st = batch_struct(hb, lambda n: hb.arrays[n].ctypes.data)
    assert lib.tw_batch_validate_host(C.byref(st)) == 0
    # skip budgets (n_out != n_in) are rejected loudly, not silently mis-solved
    p = _toy()
    p.out_start[1] = p.out_start[1][:-1]
    p.out_end[1] = p.out_end[1][:-1]
    hb2 = build_batch([p])
    st2 = batch_struct(hb2, lambda n: hb2.arrays[n].ctypes.data)
    assert lib.tw_batch_validate_host(C.byref(st2)) == -5      # the two-pass entry points; tw_skip_solve takes it
    assert b"tw_skip_solve" in lib.tw_last_error()


def test_no_device_fails_loudly(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = C.c_void_p()
    assert lib.tw_engine_create(0, C.byref(h)) == -6
    from traceweaver_b200.engine import Engine
    with pytest.raises(RuntimeError):
        Engine(0)


def test_terms_follow_reference_order():
    # hotel frontend DAG: search -> reservation -> profile plus transitive search -> profile
    s = np.arange(4, dtype=np.int64)
    p = Problem(in_start=s, in_end=s + 1, out_start=[s] * 3, out_end=[s] * 3, preds=[[], [0], [0, 1]])
    assert p.terms() == [(0, -1), (0, -2), (1, 0), (1, -2), (2, 1), (2, -2)]
    assert not p.is_primary(0, 2) and p.is_primary(1, 2)


def _mixed_blocks():
    from traceweaver_b200 import synth
    blocks = [synth.make_block("hotel_frontend", 3, 40, 100.0, seed=1),
              synth.make_block("media_nginx", 4, 25, 100.0, seed=2),
              synth.make_block("single", 2, 30, 100.0, seed=3)]
    return blocks, [blk.problem(s) for blk in blocks for s in range(blk.in_start.shape[0])]


def test_batch_slice_equals_rebuilt_batch():
    """HostBatch.slice(lo, hi) == build_batch(problems[lo:hi]) array for array (chunked solver, api.py)."""
    from traceweaver_b200.batch import build_batch, build_batch_from_blocks
    blocks, probs = _mixed_blocks()
    hb = build_batch_from_blocks(blocks)
    full = build_batch(probs)
    for k, v in full.arrays.items():
        assert np.array_equal(hb.arrays[k], v), k
    for lo, hi in ((0, 9), (0, 1), (2, 5), (3, 7), (8, 9)):
        want = build_batch(probs[lo:hi])
        for src in (hb, full):
            got = src.slice(lo, hi)
            assert got.n_problems == hi - lo
            for k, v in want.arrays.items():
                assert got.arrays[k].dtype == v.dtype, k
                assert np.array_equal(got.arrays[k], v), k


def test_trace_lists_share_the_batch_offsets():
    """truth.TraceLists derives the offset tables build_batch derives; as a batch without term tables
    its TwBatch has NULL term pointers and n_term_total = 0."""
    from traceweaver_b200.truth import TraceLists
    _, probs = _mixed_blocks()
    tl = TraceLists([dict(in_start=p.in_start, in_end=p.in_end, out_start=p.out_start, out_end=p.out_end)
                     for p in probs],
                    [np.arange(p.n_in, dtype=np.int32) for p in probs],
                    [[np.arange(len(o), dtype=np.int32) for o in p.out_start] for p in probs],
                    max(p.n_in for p in probs))
    full = build_batch(probs)
    for k in ("prob_in_off", "prob_ep_off", "prob_tuple_off", "ep_out_off"):
        assert tl.arrays[k].dtype == full.arrays[k].dtype, k
        assert np.array_equal(tl.arrays[k], full.arrays[k]), k
    st = batch_struct(tl, lambda n: tl.arrays[n].ctypes.data)
    assert st.ep_term_off is None and st.ep_pred_mask is None and st.term_src is None
    assert st.n_term_total == 0
    assert st.in_start == tl.arrays["in_start"].ctypes.data
    assert (st.n_problems, st.n_ep_total, st.n_in_total, st.n_out_total) == (
        len(probs), int(full.prob_ep_off[-1]), int(full.prob_in_off[-1]), int(full.ep_out_off[-1]))
