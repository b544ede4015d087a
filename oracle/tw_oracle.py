"""ctypes front end of oracle/libtw_oracle.so (plain-C restatement of the reference hot path).

TEST INFRASTRUCTURE ONLY: the checker, never the thing measured or shipped.  The only product
code it touches is the data-only batch descriptor (`traceweaver_b200.batch`, `_abi`), so that
oracle and engine are fed byte-identical inputs."""
import ctypes as C
import os
import subprocess

import numpy as np

from traceweaver_b200 import _abi
from traceweaver_b200.batch import HostBatch, batch_struct

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_LIB_LD = None


def build(force=False):
    so = os.path.join(HERE, "libtw_oracle.so")
    srcs = [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".c", ".h"))]
    srcs.append(os.path.join(HERE, "..", "include", "traceweaver_b200.h"))
    stale = (not os.path.exists(so)) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
    if force or stale:
        subprocess.check_call(["make", "-s", "-C", HERE, "-B", "libtw_oracle.so"])
    return so


def _declare(lib):
    """The return types of the oracle's entry points (every build of it: this one and tests/oracle_f64.py)."""
    for name in ("two_params_pass0", "two_score_problem", "two_stitch_problem", "two_assess_problem",
                 "two_delays", "two_windows_from_cuts", "two_gmm_refit_ex", "two_gmm_refit_record",
                 "two_find_assignments"):
        getattr(lib, name).restype = C.c_int
    return lib


def lib():
    global _LIB
    if _LIB is None:
        _LIB = _declare(C.CDLL(build()))
    return _LIB


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _check(rc, where):
    if rc != 0:
        raise _abi.TwError(rc, "oracle." + where)


class OracleBatch:
    """Host-pointer view of a HostBatch."""

    def __init__(self, hb: HostBatch):
        self.hb = hb
        self.struct = batch_struct(hb, lambda name: _ptr(hb.arrays[name]))

    # -- parameters --------------------------------------------------------------------------
    def params_pass0(self):
        hb = self.hb
        gauss = np.zeros((int(hb.prob_gauss_off[-1]), _abi.TW_GAUSS_REC), np.float64)
        for p in range(hb.n_problems):
            _check(lib().two_params_pass0(C.byref(self.struct), p, _ptr(hb.prob_gauss_off), _ptr(gauss)),
                   "params_pass0")
        return gauss

    def _params_struct(self, gauss=None, mix=None):
        s = _abi.TwParams()
        if mix is not None:
            s.mode = _abi.TW_PARAMS_MIXTURE
            s.mix = _ptr(mix)
        else:
            s.mode = _abi.TW_PARAMS_GAUSS_BATCHED
            s.gauss = _ptr(gauss)
        s.prob_gauss_off = _ptr(self.hb.prob_gauss_off)
        return s

    # -- scoring on undeleted lists + cuts ---------------------------------------------------
    def score(self, gauss=None, mix=None):
        hb = self.hb
        n = int(hb.prob_in_off[-1])
        nt = int(hb.prob_tuple_off[-1])
        res = dict(topk_score=np.full((n, _abi.TW_K), np.nan), topk_idx=np.full(_abi.TW_K * nt, -1, np.int32),
                   topk_cnt=np.zeros(n, np.uint8), n_feasible=np.zeros(n, np.int32), cut=np.zeros(n, np.uint8))
        out = _abi.fill(_abi.TwScoreOut, res)
        have = gauss is not None or mix is not None
        prm = self._params_struct(gauss, mix) if have else None
        for p in range(hb.n_problems):
            _check(lib().two_score_problem(C.byref(self.struct), p, C.byref(prm) if have else None, C.byref(out)),
                   "score")
        return res

    # -- one pass of the hot loop ------------------------------------------------------------
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
            _check(lib().two_stitch_problem(C.byref(self.struct), p, C.byref(prm), _ptr(cut), C.byref(out)),
                   "stitch")
        return res

    # -- the likelihood of a given assignment ------------------------------------------------
    def score_assignments(self, assign, gauss=None, mix=None):
        """two_assess_problem: score / code per in-span, prob_sum / prob_count per service (scores added in
        in-span order)."""
        hb = self.hb
        n = int(hb.prob_in_off[-1])
        res = dict(score=np.full(n, np.nan), code=np.zeros(n, np.uint8), prob_sum=np.zeros(hb.n_problems),
                   prob_count=np.zeros((hb.n_problems, _abi.TW_ASSESS_NCODES), np.int32))
        prm = self._params_struct(gauss, mix)
        assign = np.ascontiguousarray(assign, np.int32)
        for p in range(hb.n_problems):
            _check(lib().two_assess_problem(C.byref(self.struct), p, C.byref(prm), _ptr(assign),
                                            _ptr(res["score"]), _ptr(res["code"]), _ptr(res["prob_sum"]),
                                            _ptr(res["prob_count"])), "score_assignments")
        return res

    def delays(self, assign):
        hb = self.hb
        nt = int(hb.ep_term_off[-1])
        delays = np.zeros(int(hb.term_sample_off[-1]), np.float64)
        counts = np.zeros(nt, np.int32)
        assign = np.ascontiguousarray(assign, np.int32)
        for p in range(hb.n_problems):
            _check(lib().two_delays(C.byref(self.struct), p, _ptr(assign), _ptr(hb.term_sample_off),
                                    _ptr(delays), _ptr(counts)), "delays")
        return delays, counts


def windows_from_cuts(cut):
    cut = np.ascontiguousarray(cut, np.uint8)
    we = np.zeros_like(cut)
    lib().two_windows_from_cuts(len(cut), _ptr(cut), _ptr(we))
    ends = np.flatnonzero(we)
    starts = np.concatenate([[0], ends[:-1] + 1])
    return list(zip(starts.tolist(), ends.tolist()))


def _gmm_twin():
    """libtw_oracle_gmm_ld.so: the refit alone with long double accumulators (built on first use)."""
    global _LIB_LD
    if _LIB_LD is None:
        so = os.path.join(HERE, "libtw_oracle_gmm_ld.so")
        src = [os.path.join(HERE, f) for f in ("tw_oracle_gmm.c", "tw_oracle.h")]
        if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in src):
            subprocess.check_call(["make", "-s", "-C", HERE, "-B", "libtw_oracle_gmm_ld.so"])
        _LIB_LD = C.CDLL(so)
        _LIB_LD.two_gmm_refit_record.restype = C.c_int
    return _LIB_LD


GMM_REC_FIELDS = ("status", "lloyd_iter", "lloyd_strict", "relocations", "em_iter", "em_converged", "replay",
                  "lloyd_ties")


def gmm_refit(term_sample_off, delays, counts, seed_select=10, rng_skip=None, want_record=False, twin=False):
    """two_gmm_refit_record: per-term BIC-selected 1-D GMM (restated sklearn, oracle/tw_oracle_gmm.c).
    Returns (mix[n_terms, TW_MIX_REC], n_selected, max_n); with want_record also bic[n_terms, 5], the 'diag'
    BIC of each component count (+inf where that fit is not tried or raises), and rec[n_terms, 6, 8], the
    decisions of each fit (row k - 1: the 'diag' fit with k components, row 5: the final 'full' fit; columns
    GMM_REC_FIELDS).  twin: the same fit with long double accumulators."""
    L = _gmm_twin() if twin else lib()
    nt = len(counts)
    off = np.ascontiguousarray(term_sample_off, np.int64)
    delays = np.ascontiguousarray(delays, np.float64)
    counts = np.ascontiguousarray(counts, np.int32)
    mix = np.zeros((nt, _abi.TW_MIX_REC), np.float64)
    nsel = np.zeros(nt, np.int32)
    maxn = np.zeros(nt, np.int32)
    bic = np.zeros((nt, _abi.TW_GMM_MAX_COMP), np.float64) if want_record else None
    rec = np.zeros((nt, _abi.TW_GMM_MAX_COMP + 1, len(GMM_REC_FIELDS)), np.int32) if want_record else None
    skip = None if rng_skip is None else np.ascontiguousarray(rng_skip, np.uint32)
    _check(L.two_gmm_refit_record(C.c_int32(nt), _ptr(off), _ptr(delays), _ptr(counts), C.c_uint32(seed_select),
                                  _ptr(skip), _ptr(mix), _ptr(nsel), _ptr(maxn), _ptr(bic), _ptr(rec)), "gmm_refit")
    return (mix, nsel, maxn, bic, rec) if want_record else (mix, nsel, maxn)


def find_assignments(hb: HostBatch, seed_select=10, threads=1, want_topk=True):
    """two_find_assignments: the whole restated path over a batch on `threads` host threads."""
    L = lib()
    n, nt = int(hb.prob_in_off[-1]), int(hb.prob_tuple_off[-1])
    nterm = int(hb.ep_term_off[-1])
    res = dict(assign=np.full(nt, -1, np.int32), mis_rank=np.full(n, -1, np.int8), n_cand=np.zeros(n, np.int32),
               counters=np.zeros((hb.n_problems, 4), np.int32), n_cand_total=np.zeros(n, np.int32),
               mix=np.zeros((nterm, _abi.TW_MIX_REC)))
    final = _abi.fill(_abi.TwPassOut, res)            # the final pass writes no top-K lists
    if want_topk:
        res.update(topk_score=np.full((n, _abi.TW_K), np.nan), topk_idx=np.full(_abi.TW_K * nt, -1, np.int32),
                   topk_cnt=np.zeros(n, np.uint8))
    top = _abi.fill(_abi.TwScoreOut, res)
    st = batch_struct(hb, lambda name: _ptr(hb.arrays[name]))
    _check(L.two_find_assignments(C.byref(st), C.c_uint32(seed_select), C.c_int(threads), C.byref(final),
                                  C.byref(top) if want_topk else None, _ptr(res["n_cand_total"]), _ptr(res["mix"])),
           "find_assignments")
    return res
