"""ctypes front end of tests/emul/libtw_emul.so: the engine's device functions (tw_core.cuh,
tw_skip_core.cuh) compiled for the CPU and stepped sequentially (tw_emul.cpp; the request-tree analyses in
tw_emul_critical.cpp and tw_emul_confidence.cpp).  Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.tw_oracle import OracleBatch, _ptr, _check
from traceweaver_b200 import _abi
from traceweaver_b200.batch import HostBatch, batch_struct

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        subprocess.check_call(["make", "-s", "-C", HERE, "libtw_emul.so"], stderr=subprocess.DEVNULL)
        _LIB = C.CDLL(os.path.join(HERE, "libtw_emul.so"))
    return _LIB


class EmulBatch(OracleBatch):
    """Same interface as OracleBatch, but running the engine's own per-thread code.

    table_cap: term-table slots available per in-span (0 forces the per-leaf path).
    light_combos: in-spans with more candidate combinations than this use the lane-parallel path (-1: never)."""

    W = 2              # bitmap words per (in-span, ep): the narrow kernel's width
    node_limit = 0

    def __init__(self, hb, table_cap=4096, light_combos=-1):
        super().__init__(hb)
        self.table_cap = int(table_cap)
        self.light_combos = int(light_combos)

    def _paths(self):
        return C.c_int(self.table_cap), C.c_longlong(self.light_combos)

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
                                           C.byref(out), W, C.byref(ov), *self._paths()), "emul.score")
            if ov.value:  # the engine re-runs overflowing tiles with the wide kernel
                W = 64
                _check(lib().twe_score_problem(C.byref(self.struct), p, C.byref(prm) if have else None,
                                               C.byref(out), W, C.byref(ov), *self._paths()), "emul.score")
                if ov.value:  # a feasible candidate at offset >= 2048: what the redo kernel reports
                    raise _abi.TwError(_abi.TW_ERR_RANGE_LIMIT, "emul.score")
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
                                            C.c_longlong(self.node_limit), *self._paths()), "emul.stitch")
        return res

    def score_assignments(self, assign, gauss=None, mix=None, top=None):
        """k_assess stepped on the CPU: score / code (/ margin with `top`, a final top-K) per in-span,
        prob_sum / prob_count per service in the kernels' summation order."""
        hb = self.hb
        n, P = int(hb.prob_in_off[-1]), hb.n_problems
        res = dict(score=np.full(n, -7.0), code=np.full(n, 99, np.uint8), margin=np.full(n, -7.0),
                   prob_sum=np.zeros(P), prob_count=np.zeros((P, _abi.TW_ASSESS_NCODES), np.int32))
        prm = self._params_struct(gauss, mix)
        assign = np.ascontiguousarray(assign, np.int32)
        tk = None
        if top is not None:
            keep = {k: np.ascontiguousarray(top[k]) for k in ("topk_score", "topk_idx", "topk_cnt")}
            tk = _abi.fill(_abi.TwScoreOut, keep)
        for p in range(P):
            _check(lib().twe_assess_problem(C.byref(self.struct), p, C.byref(prm), _ptr(assign),
                                            C.byref(tk) if tk is not None else None, _ptr(res["score"]),
                                            _ptr(res["code"]), _ptr(res["margin"]), _ptr(res["prob_sum"]),
                                            _ptr(res["prob_count"])), "emul.assess")
        if top is None:
            del res["margin"]
        return res


def _skip_service(in_start, in_end, out_start, out_end, preds, wins, counts, pair, budgets):
    """One cache-mode service through the product's own marshalling (traceweaver_b200.skipmode.marshal) with
    host pointers: the callee lists' sort order, the batch and the skip descriptor's arrays."""
    from traceweaver_b200 import skipmode
    order, s_start, s_end = skipmode.sort_partitions(out_start, out_end)
    hb, host = skipmode.marshal(np.ascontiguousarray(in_start, np.int64), np.ascontiguousarray(in_end, np.int64),
                                s_start, s_end, order, preds, wins, counts, pair, budgets)
    return order, OracleBatch(hb), host


def skip_solve(in_start, in_end, out_start, out_end, preds, wins, counts, pair, budgets, node_limit=2000000):
    """k_skip's body (tw_skip_core.cuh) stepped on the CPU.  Results in the caller's list order."""
    from traceweaver_b200 import skipmode
    order, ob, host = _skip_service(in_start, in_end, out_start, out_end, preds, wins, counts, pair, budgets)
    E, n = len(out_start), len(in_start)
    nt = n * E
    out = dict(assign=np.full(nt, -9, np.int32), mis_rank=np.full(n, -9, np.int8), n_cand=np.zeros(n, np.int32),
               topk_score=np.full((n, _abi.TW_K), np.nan), topk_idx=np.full(_abi.TW_K * nt, -1, np.int32),
               topk_cnt=np.zeros(n, np.uint8), counters=np.zeros((1, 4), np.int32),
               top2_score=np.full((n, _abi.TW_K), np.nan), top2_idx=np.full(_abi.TW_K * nt, -1, np.int32),
               top2_cnt=np.zeros(n, np.uint8), cut=np.zeros(n, np.uint8))
    sd = _abi.fill(_abi.TwSkipDesc, host)
    so = _abi.fill(_abi.TwSkipOut, out)
    _check(lib().twe_skip_solve(C.byref(ob.struct), C.byref(sd), C.byref(so), C.c_longlong(node_limit)),
           "emul.skip_solve")
    return skipmode.to_caller_order(out, order, n, E)


def skip_score(in_start, in_end, out_start, out_end, preds, assign, wins, counts, pair, budgets, top2=None):
    """k_skip_assess stepped on the CPU over one cache-mode service; assign [E, n] and top2 (top2_score [n, K],
    top2_idx [n, K, E], top2_cnt [n]) in the caller's list positions.  Returns score / code (/ margin) [n],
    service_score and service_codes in the kernels' summation order."""
    from traceweaver_b200 import skipmode
    order, ob, host = _skip_service(in_start, in_end, out_start, out_end, preds, wins, counts, pair, budgets)
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
    _check(lib().twe_skip_assess_problem(C.byref(ob.struct), 0, C.byref(sd), _ptr(a),
                                         C.byref(tk) if tk is not None else None, _ptr(res["score"]),
                                         _ptr(res["code"]), _ptr(res["margin"]), _ptr(res["prob_sum"]),
                                         _ptr(res["prob_count"])), "emul.skip_assess")
    out = dict(score=res["score"], code=res["code"], service_score=float(res["prob_sum"][0]),
               service_codes=res["prob_count"][0])
    if top2 is not None:
        out["margin"] = res["margin"]
    return out


def _host_struct(hb):
    a = {k: np.ascontiguousarray(v) for k, v in hb.arrays.items()}
    return a, batch_struct(HostBatch(problems=hb.problems, arrays=a), lambda k: a[k].ctypes.data)


def critical_paths(hb, assign, in_caller, root, slow_us, levels=0):
    """The critical-path walk with the kernels' per-node steps, stepped on the CPU; the join's roots come in.
    levels: the level launches, the last of them walking what lies below it (cp_tail_walk); 0: until nothing
    is left."""
    a, st = _host_struct(hb)
    times = _abi.fill(_abi.TwTimesF64, a) if hb.float_times else None
    n_in, n = int(hb.prob_in_off[-1]), int(hb.prob_in_off[-1]) + int(hb.ep_out_off[-1])
    P, n_ep = hb.n_problems, int(hb.prob_ep_off[-1])
    out = dict(on_path=np.zeros(n, np.uint8), self_us=np.zeros(n), culprit=np.zeros(n_in, np.int32),
               server_us=np.zeros((P, 2)), server_visits=np.zeros((P, 2), np.int32), call_us=np.zeros((n_ep, 2)),
               requests=np.zeros(2, np.int32))
    links = [np.ascontiguousarray(x, np.int32).reshape(-1) for x in (assign, in_caller, root)]
    rc = lib().twe_critical_paths(C.byref(st), C.byref(times) if times is not None else None,
                                  *[_ptr(x) for x in links], C.c_double(slow_us), C.c_int(levels),
                                  *[_ptr(out[k]) for k in ("on_path", "self_us", "culprit", "server_us",
                                                           "server_visits", "call_us", "requests")])
    assert rc == 0
    out["root"] = links[2]
    return out


def request_confidence(hb, assign, root, score, code, topk):
    """The step, the per-request passes and the fixed-order sums of tw_confidence.cu stepped on the CPU; the
    join's roots come in.  Returns the arrays and the return code."""
    _, st = _host_struct(hb)
    n_in, P = int(hb.prob_in_off[-1]), hb.n_problems
    ins = [np.ascontiguousarray(np.asarray(x, t).reshape(-1)) for x, t in
           ((assign, np.int32), (root, np.int32), (score, np.float64), (code, np.uint8),
            (topk["topk_score"], np.float64), (topk["topk_idx"], np.int32), (topk["topk_cnt"], np.uint8))]
    out = dict(p=np.zeros(n_in), ell=np.zeros(n_in), q=np.zeros(n_in, np.int64), decisions=np.zeros(n_in, np.int32),
               zero=np.zeros(n_in, np.int32), log_conf=np.zeros(n_in, np.int64), conf=np.zeros(n_in),
               weakest=np.zeros(n_in, np.int32), weakest_p=np.zeros(n_in), est_accuracy=np.zeros(P),
               requests=np.zeros(1, np.int32), expected_exact=np.zeros(1))
    order = ("p", "ell", "q", "decisions", "zero", "log_conf", "conf", "weakest", "weakest_p", "est_accuracy",
             "requests", "expected_exact")
    rc = lib().twe_request_confidence(C.byref(st), *[_ptr(x) for x in ins], *[_ptr(out[k]) for k in order])
    return out, rc


def _elementwise(name, v):
    v = np.ascontiguousarray(v, np.float64)
    got = np.zeros_like(v)
    getattr(lib(), name)(C.c_int64(len(v)), _ptr(v), _ptr(got))
    return got


def conf_exp(d):
    """tw_core.cuh's conf_exp of every element of d, on the CPU."""
    return _elementwise("twe_conf_exp", d)


def conf_log(x):
    """tw_core.cuh's conf_log of every element of x, on the CPU."""
    return _elementwise("twe_conf_log", x)


def first_centre(u, n):
    """tw_core.cuh's first_centre (the refit's first k-means++ centre) of every (u, n) pair, on the CPU."""
    u, n = np.broadcast_arrays(np.asarray(u, np.float64), np.asarray(n, np.int32))
    u, n = np.ascontiguousarray(u).reshape(-1), np.ascontiguousarray(n).reshape(-1)
    out = np.zeros(len(u), np.int32)
    lib().twe_first_centre(C.c_int64(len(u)), _ptr(u), _ptr(n), _ptr(out))
    return out
