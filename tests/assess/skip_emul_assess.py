"""k_skip_assess stepped on the CPU (tests/assess/tw_emul_skip_assess.cpp over the engine's own
skip_assess_in_span).  TEST INFRASTRUCTURE ONLY.  Compiled into a temporary directory keyed by the hash of
its sources (assess_backends._build), so the tree is never written."""
import ctypes as C

import numpy as np

from assess_backends import _LIBS, _build, _read
from oracle.tw_oracle import _check, _ptr
from traceweaver_b200 import _abi

SOURCES = ("traceweaver_b200/csrc/tw_core.cuh", "traceweaver_b200/csrc/tw_skip_core.cuh", "include/traceweaver_b200.h",
           "tests/assess/tw_emul_assess.cpp", "tests/assess/tw_emul_skip_assess.cpp")


def _lib():
    if "emul_skip" not in _LIBS:
        files = {rel: _read(rel) for rel in SOURCES}
        cmd = lambda d, out: ["g++", "-O2", "-fPIC", "-std=c++17", "-Wall", "-ffp-contract=off", "-shared", "-x", "c++",
                              "-o", out, f"{d}/tests/assess/tw_emul_skip_assess.cpp", "-lm"]
        lib = _build("emul_skip", files, cmd)
        lib.twe_skip_assess_problem.restype = C.c_int
        _LIBS["emul_skip"] = lib
    return _LIBS["emul_skip"]


def emul_skip_score(in_start, in_end, out_start, out_end, preds, assign, wins, counts, pair, budgets, top2=None):
    """One cache-mode service marshalled as skipmode does it; assign [E, n] and top2 (top2_score [n, K],
    top2_idx [n, K, E], top2_cnt [n]) in the caller's list positions.  Returns score / code (/ margin) [n],
    service_score and service_codes in the kernels' summation order."""
    from traceweaver_b200 import skipmode
    from traceweaver_b200.batch import batch_struct
    in_start = np.ascontiguousarray(in_start, np.int64)
    in_end = np.ascontiguousarray(in_end, np.int64)
    order, s_start, s_end = skipmode.sort_partitions(out_start, out_end)
    hb, host = skipmode.marshal(in_start, in_end, s_start, s_end, order, preds, wins, counts, pair, budgets)
    n = len(in_start)
    a = np.ascontiguousarray(skipmode.to_sorted_order(assign, order, False).reshape(-1))
    res = dict(score=np.full(n, -7.0), code=np.full(n, 99, np.uint8), margin=np.full(n, -7.0), prob_sum=np.zeros(1),
               prob_count=np.zeros((1, _abi.TW_SKIP_ASSESS_NCODES), np.int32))
    tk = None
    if top2 is not None:
        keep = dict(top2_score=np.ascontiguousarray(top2["top2_score"], np.float64),
                    top2_idx=np.ascontiguousarray(skipmode.to_sorted_order(top2["top2_idx"], order, True).reshape(-1)),
                    top2_cnt=np.ascontiguousarray(top2["top2_cnt"], np.uint8))
        tk = _abi.fill(_abi.TwSkipOut, keep)
    sd = _abi.fill(_abi.TwSkipDesc, host)
    st = batch_struct(hb, lambda name: _ptr(hb.arrays[name]))
    _check(_lib().twe_skip_assess_problem(C.byref(st), 0, C.byref(sd), _ptr(a), C.byref(tk) if tk is not None else None,
                                          _ptr(res["score"]), _ptr(res["code"]), _ptr(res["margin"]),
                                          _ptr(res["prob_sum"]), _ptr(res["prob_count"])), "emul.skip_assess")
    out = dict(score=res["score"], code=res["code"], service_score=float(res["prob_sum"][0]),
               service_codes=res["prob_count"][0])
    if top2 is not None:
        out["margin"] = res["margin"]
    return out
