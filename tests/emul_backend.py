"""ctypes front end of tests/emul/libtw_emul.so: the engine's device functions (tw_core.cuh)
compiled for the CPU and stepped sequentially.  Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.tw_oracle import OracleBatch, _ptr, _check
from traceweaver_b200 import _abi

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-s", "-C", HERE, "libtw_emul.so"], stderr=subprocess.DEVNULL)
        _LIB = C.CDLL(os.path.join(HERE, "libtw_emul.so"))
    return _LIB


def set_table_cap(cap):
    """Term-table slots available per in-span (0 forces the per-leaf path)."""
    lib().twe_set_table_cap(int(cap))


def set_light_combos(c):
    """In-spans with more candidate combinations than this use the lane-parallel path (-1: never)."""
    lib().twe_set_light_combos(C.c_longlong(int(c)))


class EmulBatch(OracleBatch):
    """Same interface as OracleBatch, but running the engine's own per-thread code."""

    W = 2              # bitmap words per (in-span, ep): the narrow kernel's width
    node_limit = 0

    def score(self, gauss=None, mix=None):
        hb = self.hb
        n = int(hb.prob_in_off[-1])
        nt = int(hb.prob_tuple_off[-1])
        res = dict(topk_score=np.full((n, _abi.TW_K), np.nan), topk_idx=np.full(_abi.TW_K * nt, -1, np.int32),
                   topk_cnt=np.zeros(n, np.uint8), n_feasible=np.zeros(n, np.int32), cut=np.zeros(n, np.uint8))
        out = _abi.fill(_abi.TwScoreOut, res)
        have = gauss is not None or mix is not None
        prm = self._params_struct(gauss, mix) if have else None
        self.overflow = []
        for p in range(hb.n_problems):
            ov = C.c_int(0)
            W = self.W
            _check(lib().twe_score_problem(C.byref(self.struct), p, C.byref(prm) if have else None,
                                           C.byref(out), W, C.byref(ov)), "emul.score")
            if ov.value:  # the engine re-runs overflowing tiles with the wide kernel
                W = 64
                _check(lib().twe_score_problem(C.byref(self.struct), p, C.byref(prm) if have else None,
                                               C.byref(out), W, C.byref(ov)), "emul.score")
                assert not ov.value
            self.overflow.append(W)
        return res

    def stitch(self, cut, gauss=None, mix=None, want_topk=True):
        hb = self.hb
        n = int(hb.prob_in_off[-1])
        nt = int(hb.prob_tuple_off[-1])
        res = dict(assign=np.full(nt, -1, np.int32), mis_rank=np.full(n, -1, np.int8),
                   n_cand=np.zeros(n, np.int32),
                   topk_score=np.full((n, _abi.TW_K), np.nan) if want_topk else None,
                   topk_idx=np.full(_abi.TW_K * nt, -1, np.int32) if want_topk else None,
                   topk_cnt=np.zeros(n, np.uint8) if want_topk else None,
                   counters=np.zeros((hb.n_problems, 4), np.int32))
        out = _abi.fill(_abi.TwPassOut, res)
        prm = self._params_struct(gauss, mix)
        cut = np.ascontiguousarray(cut, np.uint8)
        for p in range(hb.n_problems):
            _check(lib().twe_stitch_problem(C.byref(self.struct), p, C.byref(prm), _ptr(cut), C.byref(out),
                                            C.c_longlong(self.node_limit)), "emul.stitch")
        return res


def skip_solve(in_start, in_end, out_start, out_end, preds, wins, counts, pair, budgets, node_limit=2000000):
    """k_skip's body (tw_skip_core.cuh) stepped on the CPU, fed through the product's own marshalling
    (traceweaver_b200.skipmode.marshal) with host pointers.  Results in the caller's list order."""
    from traceweaver_b200 import skipmode
    from traceweaver_b200.batch import batch_struct
    in_start = np.ascontiguousarray(in_start, np.int64)
    in_end = np.ascontiguousarray(in_end, np.int64)
    order, s_start, s_end = skipmode.sort_partitions(out_start, out_end)
    hb, host = skipmode.marshal(in_start, in_end, s_start, s_end, order, preds, wins, counts, pair, budgets)
    E, n = len(out_start), len(in_start)
    nt = n * E
    out = dict(assign=np.full(nt, -9, np.int32), mis_rank=np.full(n, -9, np.int8), n_cand=np.zeros(n, np.int32),
               topk_score=np.full((n, _abi.TW_K), np.nan), topk_idx=np.full(_abi.TW_K * nt, -1, np.int32),
               topk_cnt=np.zeros(n, np.uint8), counters=np.zeros((1, 4), np.int32),
               top2_score=np.full((n, _abi.TW_K), np.nan), top2_idx=np.full(_abi.TW_K * nt, -1, np.int32),
               top2_cnt=np.zeros(n, np.uint8), cut=np.zeros(n, np.uint8))
    sd = _abi.fill(_abi.TwSkipDesc, host)
    so = _abi.fill(_abi.TwSkipOut, out)
    st = batch_struct(hb, lambda name: _ptr(hb.arrays[name]))
    L = lib()
    L.twe_skip_solve.restype = C.c_int
    _check(L.twe_skip_solve(C.byref(st), C.byref(sd), C.byref(so), C.c_longlong(node_limit)), "emul.skip_solve")
    return skipmode.to_caller_order(out, order, n, E)
