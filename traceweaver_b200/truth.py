"""Ground truth, invocation order and accuracy on the device (SURVEY.md §8 row f-2): thin wrappers
around tw_ground_truth / tw_find_order / tw_accuracy (csrc/tw_truth.cu), which replace
utils.GetGroundTruth (helpers/utils.py:22-32), the pruning loop of FindOrder (executor.py:214-285) and
the accuracy helpers (helpers/utils.py:62-145) by joins on densely numbered trace ids."""
import ctypes as C

import numpy as np
import torch

from . import _abi, _lib
from .batch import batch_struct, offset_tables
from .engine import _p, _to_device


class TraceLists:
    """Offset tables + span arrays of a list of services whose callees are in ANY order (the order is
    what FindOrder derives) plus the trace number of every span.  probs[p] = dict(in_start, in_end,
    out_start=[per callee], out_end=[...]); in_trace[p]: int32 [n_in]; out_trace[p]: per callee int32."""

    def __init__(self, probs, in_trace, out_trace, n_traces):
        a = offset_tables([len(q["in_start"]) for q in probs], [len(q["out_start"]) for q in probs],
                          [len(o) for q in probs for o in q["out_start"]])
        cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0, dt), dt)
        a["in_start"] = cat([q["in_start"] for q in probs], np.int64)
        a["in_end"] = cat([q["in_end"] for q in probs], np.int64)
        a["out_start"] = cat([o for q in probs for o in q["out_start"]], np.int64)
        a["out_end"] = cat([o for q in probs for o in q["out_end"]], np.int64)
        a["in_trace"] = cat(list(in_trace), np.int32)
        a["out_trace"] = cat([o for q in out_trace for o in q], np.int32)
        lo = np.array([int(t.min()) if len(t) else 0 for t in in_trace], np.int32)
        hi = np.array([int(t.max()) if len(t) else -1 for t in in_trace], np.int32)
        a["prob_trace_lo"] = lo
        a["prob_trace_n"] = (hi - lo + 1).astype(np.int32)
        self.arrays = a
        self.n_problems = len(probs)
        self.n_traces = int(n_traces)
        self.d = None

    @classmethod
    def from_host_batch(cls, hb, in_trace, n_traces):
        """For tw_accuracy on a solved batch: offsets of `hb`, trace number per in-span (global array)."""
        self = cls.__new__(cls)
        a = {k: hb.arrays[k] for k in ("prob_in_off", "prob_ep_off", "prob_tuple_off", "ep_out_off", "in_start",
                                       "in_end", "out_start", "out_end")}
        a["in_trace"] = None if in_trace is None else np.ascontiguousarray(in_trace, np.int32)
        self.arrays = a
        self.n_problems = hb.n_problems
        self.n_traces = int(n_traces)
        self.d = None
        return self

    def upload(self, device, resident=None):
        if self.d is None:
            self.d = _to_device(self.arrays, device, resident)
        return self.d


def _structs(engine, tl: TraceLists, resident=None):
    d = tl.upload(engine.device, resident)
    dev = batch_struct(tl, lambda n: d[n].data_ptr())
    host = batch_struct(tl, lambda n: tl.arrays[n].ctypes.data)
    return d, dev, host


def ground_truth(engine, tl: TraceLists):
    """truth[tuple_off[p] + e*n_p + i] (device int32): position of in-span i's child in callee e's list."""
    d, dev, host = _structs(engine, tl)
    keys = _abi.fill(_abi.TwTraceKeys, d, n_traces=tl.n_traces)
    truth = torch.empty(int(tl.arrays["prob_tuple_off"][-1]), dtype=torch.int32, device=engine.device)
    _lib.check(engine.lib.tw_ground_truth(engine.h, C.byref(dev), C.byref(host), C.byref(keys),
                                          C.c_void_p(tl.arrays["prob_trace_n"].ctypes.data), _p(truth), engine.stream),
               "tw_ground_truth")
    return truth


def find_order(engine, tl: TraceLists, truth):
    """Per callee a (global ep index): bit b set = edge a -> b violated by some trace (numpy uint32)."""
    d, dev, host = _structs(engine, tl)
    viol = torch.empty(int(tl.arrays["prob_ep_off"][-1]), dtype=torch.int32, device=engine.device)
    _lib.check(engine.lib.tw_find_order(engine.h, C.byref(dev), C.byref(host), _p(truth), _p(viol), engine.stream),
               "tw_find_order")
    return viol.cpu().numpy().view(np.uint32)


def accuracy(engine, tl: TraceLists, truth, assign, topk_idx=None, topk_cnt=None, prob_first=None, resident=None):
    """AccuracyForService / TopKAccuracyForService per service and the two end-to-end accuracies
    (helpers/utils.py:62-145).  truth / assign / topk_*: device tensors in the engine's layouts."""
    d, dev, host = _structs(engine, tl, resident)
    P = tl.n_problems
    per = torch.empty((P, 2), dtype=torch.int64, device=engine.device)
    e2e = torch.empty(4, dtype=torch.int64, device=engine.device)
    pf = None if prob_first is None else _to_device(dict(pf=np.asarray(prob_first, np.uint8)), engine.device)["pf"]
    in_trace = d.get("in_trace")
    _lib.check(engine.lib.tw_accuracy(engine.h, C.byref(dev), C.byref(host), _p(truth), _p(assign), _p(topk_idx),
                                      _p(topk_cnt), _p(in_trace), tl.n_traces if in_trace is not None else 0, _p(pf),
                                      _p(per), _p(e2e), engine.stream), "tw_accuracy")
    per = per.cpu().numpy()
    e2e = e2e.cpu().numpy()
    n_in = np.diff(tl.arrays["prob_in_off"])
    return dict(correct=per[:, 0], topk_correct=per[:, 1], n_in=n_in,
                service_accuracy=per[:, 0] / np.maximum(n_in, 1), service_topk_accuracy=per[:, 1] / np.maximum(n_in, 1),
                traces=int(e2e[0]), traces_correct=int(e2e[1]), traces_topk_correct=int(e2e[3]),
                e2e_accuracy=(e2e[1] / e2e[0]) if e2e[0] else None,
                e2e_topk_accuracy=(e2e[3] / e2e[2]) if e2e[2] else None)
