"""Thin Python handle on the CUDA engine: device buffers as torch tensors (plumbing only), every
compute step is a call through the C ABI of libtw_b200.so."""
import ctypes as C

import numpy as np
import torch

from . import _abi, _lib
from .batch import SPAN_ARRAYS, HostBatch, batch_struct


def _to_device(arrays, device, resident=None, pinned=()):
    """Device tensors of a name -> host array mapping; the one way host arrays reach the device.
    None entries are left out, a name in `resident` adopts the tensor given there (already on the
    device), names in `pinned` go through page-locked staging (asynchronous copy).  uint32 arrays
    travel as int32: torch has no uint32 tensors, the kernels read the bits."""
    d = {}
    for name, a in arrays.items():
        if a is None:
            continue
        if resident and name in resident:
            d[name] = resident[name]
            continue
        if a.dtype == np.uint32:
            a = a.view(np.int32)
        t = torch.from_numpy(np.ascontiguousarray(a))
        if name in pinned:
            t = t.pin_memory()
        d[name] = t.to(device, non_blocking=name in pinned)
    return d


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class Params:
    """Delay-distribution parameters of one pass (tw_params)."""

    def __init__(self, mode, table, prob_gauss_off):
        self.mode = mode
        self.table = table
        self.prob_gauss_off = prob_gauss_off

    def struct(self):
        s = _abi.TwParams()
        s.mode = self.mode
        s.prob_gauss_off = self.prob_gauss_off.data_ptr()
        if self.mode == _abi.TW_PARAMS_GAUSS_BATCHED:
            s.gauss = self.table.data_ptr()
        else:
            s.mix = self.table.data_ptr()
        return s


class Engine:
    def __init__(self, device=0):
        if not torch.cuda.is_available():
            raise RuntimeError("traceweaver_b200 needs a CUDA device (H100, sm_90a); there is no CPU path")
        self.lib = _lib.load()
        self.device = torch.device("cuda", device)
        h = C.c_void_p()
        torch.cuda.set_device(self.device)
        _lib.check(self.lib.tw_engine_create(device, C.byref(h)), "tw_engine_create")
        self.h = h
        self.hb = None
        self.d = {}

    def close(self):
        if getattr(self, "h", None):
            self.lib.tw_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # -- binding ---------------------------------------------------------------------------------
    def bind(self, hb: HostBatch, device_arrays=None, pinned=False):
        """Upload (or adopt) the batch arrays and bind them.  `device_arrays`: dict of tensors
        already resident on the device for the four span arrays.  A batch with float64 span arrays
        (fractional microseconds) is bound through tw_engine_bind_f64."""
        self.hb = hb
        self.d = d = _to_device(hb.arrays, self.device, device_arrays, SPAN_ARRAYS if pinned else ())
        self.dev_struct = batch_struct(hb, lambda n: d[n].data_ptr())
        self.host_struct = batch_struct(hb, lambda n: hb.arrays[n].ctypes.data)
        if hb.float_times:
            self.times_struct = _abi.fill(_abi.TwTimesF64, d)
            _lib.check(self.lib.tw_engine_bind_f64(self.h, C.byref(self.dev_struct), C.byref(self.host_struct),
                                                   C.byref(self.times_struct), self.stream), "tw_engine_bind_f64")
        else:
            _lib.check(self.lib.tw_engine_bind(self.h, C.byref(self.dev_struct), C.byref(self.host_struct),
                                               self.stream), "tw_engine_bind")
        self.n_in = int(hb.prob_in_off[-1])
        self.n_tuple = int(hb.prob_tuple_off[-1])
        return self

    def prepare(self):
        """tw_prepare: prev-index scan + end-time sort (part of the path, once per batch)."""
        _lib.check(self.lib.tw_prepare(self.h, self.stream), "tw_prepare")

    def status(self):
        _lib.check(self.lib.tw_engine_status(self.h, self.stream), "tw_engine_status")

    def launch_count(self):
        return int(self.lib.tw_engine_launch_count(self.h))

    def _tile_stats(self):
        nt, nr = C.c_int64(0), C.c_int64(0)
        _lib.check(self.lib.tw_engine_tile_stats(self.h, C.byref(nt), C.byref(nr), self.stream), "tw_engine_tile_stats")
        return int(nt.value), int(nr.value)

    def tile_count(self):
        return self._tile_stats()[0]

    def redo_tile_count(self):
        """Scoring tiles the last score() handed to the sequential kernel (syncs the stream)."""
        return self._tile_stats()[1]

    # -- kernels ---------------------------------------------------------------------------------
    def params_pass0(self) -> Params:
        n_rec = int(self.hb.prob_gauss_off[-1])
        gauss = torch.empty((n_rec, _abi.TW_GAUSS_REC), dtype=torch.float64, device=self.device)
        _lib.check(self.lib.tw_params_pass0(self.h, _p(self.d["prob_gauss_off"]), _p(gauss), self.stream),
                   "tw_params_pass0")
        return Params(_abi.TW_PARAMS_GAUSS_BATCHED, gauss, self.d["prob_gauss_off"])

    def params_from_host(self, gauss=None, mix=None) -> Params:
        if mix is not None:
            t = _to_device(dict(mix=np.asarray(mix, np.float64).reshape(-1, _abi.TW_MIX_REC)), self.device)
            return Params(_abi.TW_PARAMS_MIXTURE, t["mix"], self.d["prob_gauss_off"])
        t = _to_device(dict(gauss=np.asarray(gauss, np.float64).reshape(-1, _abi.TW_GAUSS_REC)), self.device)
        return Params(_abi.TW_PARAMS_GAUSS_BATCHED, t["gauss"], self.d["prob_gauss_off"])

    def score(self, params: Params = None, out=None, want_used=False, keep_windows=False):
        """tw_score_topk.  want_used: also emit the candidate maps tw_stitch's fast path needs.
        keep_windows: `out` already holds cut / used maps from an earlier call on this batch (they
        depend on the span arrays only); only the top-K lists are produced."""
        dev = self.device
        n, nt = self.n_in, self.n_tuple
        if out is None:
            out = {}
        if want_used:
            out.setdefault("used_lo", torch.empty(nt, dtype=torch.int32, device=dev))
            out.setdefault("used_bits", torch.empty(2 * nt, dtype=torch.int32, device=dev))
            out.setdefault("used_wide", torch.empty(n, dtype=torch.uint8, device=dev))
        out.setdefault("n_feasible", torch.empty(n, dtype=torch.int32, device=dev))
        out.setdefault("cut", torch.empty(n, dtype=torch.uint8, device=dev))
        if params is not None:
            out.setdefault("topk_score", torch.empty((n, _abi.TW_K), dtype=torch.float64, device=dev))
            out.setdefault("topk_idx", torch.empty(_abi.TW_K * nt, dtype=torch.int32, device=dev))
            out.setdefault("topk_cnt", torch.empty(n, dtype=torch.uint8, device=dev))
        s = _abi.fill(_abi.TwScoreOut, out, flags=_abi.TW_SCORE_KEEP_WINDOWS if keep_windows else 0)
        ps = params.struct() if params is not None else None
        _lib.check(self.lib.tw_score_topk(self.h, C.byref(ps) if ps is not None else None, C.byref(s),
                                          self.stream), "tw_score_topk")
        return out

    def stitch(self, params: Params, cut, want_topk=False, out=None, undeleted=None):
        """tw_stitch.  undeleted: result of score(params, want_used=True) with the SAME params; lets
        the kernel adopt those top-K lists wherever no candidate has been taken (identical result)."""
        dev = self.device
        n, nt = self.n_in, self.n_tuple
        if out is None:
            out = {}
        out.setdefault("assign", torch.empty(nt, dtype=torch.int32, device=dev))
        out.setdefault("mis_rank", torch.empty(n, dtype=torch.int8, device=dev))
        out.setdefault("n_cand", torch.empty(n, dtype=torch.int32, device=dev))
        out.setdefault("counters", torch.zeros((self.hb.n_problems, 4), dtype=torch.int32, device=dev))
        if want_topk:
            out.setdefault("topk_score", torch.empty((n, _abi.TW_K), dtype=torch.float64, device=dev))
            out.setdefault("topk_idx", torch.empty(_abi.TW_K * nt, dtype=torch.int32, device=dev))
            out.setdefault("topk_cnt", torch.empty(n, dtype=torch.uint8, device=dev))
        s = _abi.fill(_abi.TwPassOut, out)
        ps = params.struct()
        und = _abi.fill(_abi.TwScoreOut, undeleted) if undeleted is not None else None
        _lib.check(self.lib.tw_stitch(self.h, C.byref(ps), _p(cut), C.byref(und) if und is not None else None,
                                      C.byref(s), self.stream), "tw_stitch")
        return out

    def score_assignments(self, params: Params, assign, final_topk=None):
        """tw_score_assignments: the likelihood of a given assignment (tw_pass_out.assign layout, device
        int32) under `params`.  Device tensors: score / code [n_in] (code: TW_ASSESS_*, score NaN unless
        code 0), prob_sum [P] (sum of the scored in-spans' scores per service), prob_count [P,
        TW_ASSESS_NCODES]; with `final_topk` (a score() result under the same params) also margin [n_in]."""
        dev, n, P = self.device, self.n_in, self.hb.n_problems
        out = dict(score=torch.empty(n, dtype=torch.float64, device=dev),
                   code=torch.empty(n, dtype=torch.uint8, device=dev),
                   prob_sum=torch.empty(P, dtype=torch.float64, device=dev),
                   prob_count=torch.empty((P, _abi.TW_ASSESS_NCODES), dtype=torch.int32, device=dev))
        top = None
        if final_topk is not None:
            out["margin"] = torch.empty(n, dtype=torch.float64, device=dev)
            top = _abi.fill(_abi.TwScoreOut, {k: final_topk[k] for k in ("topk_score", "topk_idx", "topk_cnt")})
        ps = params.struct()
        _lib.check(self.lib.tw_score_assignments(self.h, C.byref(ps), _p(assign), C.byref(top) if top is not None else None,
                                                 _p(out["score"]), _p(out["code"]), _p(out.get("margin")),
                                                 _p(out["prob_sum"]), _p(out["prob_count"]), self.stream),
                   "tw_score_assignments")
        return out

    def gmm_refit(self, delays, counts, seed_select=10, prob_base_skip=None, term_order=None, want_selected=False):
        """tw_gmm_refit: BIC-selected 1-D GMM per term on the device -> mixture Params."""
        nt = int(self.hb.ep_term_off[-1])
        mix = torch.empty((nt, _abi.TW_MIX_REC), dtype=torch.float64, device=self.device)
        nsel = torch.empty(nt, dtype=torch.int32, device=self.device) if want_selected else None
        _lib.check(self.lib.tw_gmm_refit(self.h, _p(self.d["term_sample_off"]), _p(delays), _p(counts),
                                         C.c_uint32(seed_select), _p(prob_base_skip), _p(term_order), _p(mix),
                                         _p(nsel), self.stream), "tw_gmm_refit")
        prm = Params(_abi.TW_PARAMS_MIXTURE, mix, self.d["prob_gauss_off"])
        return (prm, nsel) if want_selected else prm

    def gmm_stream_draws(self, delays, counts):
        """tw_gmm_stream_draws: per-problem random_sample() consumption of a model-selection pass."""
        out = torch.empty(self.hb.n_problems, dtype=torch.int32, device=self.device)
        _lib.check(self.lib.tw_gmm_stream_draws(self.h, _p(self.d["term_sample_off"]), _p(delays), _p(counts),
                                                _p(out), self.stream), "tw_gmm_stream_draws")
        return out

    def gmm_work(self, reset=False):
        """EM sample-component evaluations since the last reset (tw_gmm_work; syncs the device)."""
        v = C.c_uint64(0)
        _lib.check(self.lib.tw_gmm_work(self.h, C.byref(v), 1 if reset else 0), "tw_gmm_work")
        return int(v.value)

    def fp64_peak_tflops(self):
        """Measured dense FP64 FMA rate of this device (tw_measure_fp64_peak)."""
        v = C.c_double(0.0)
        _lib.check(self.lib.tw_measure_fp64_peak(self.h, C.byref(v), self.stream), "tw_measure_fp64_peak")
        return float(v.value)

    def delays(self, assign):
        hb = self.hb
        delays = torch.empty(int(hb.term_sample_off[-1]), dtype=torch.float64, device=self.device)
        counts = torch.empty(int(hb.ep_term_off[-1]), dtype=torch.int32, device=self.device)
        _lib.check(self.lib.tw_delays(self.h, _p(assign), _p(self.d["term_sample_off"]), _p(delays), _p(counts),
                                      self.stream), "tw_delays")
        return delays, counts
