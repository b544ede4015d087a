"""ctypes mirror of include/traceweaver_b200.h (the C ABI of the engine).

Field order and widths must match the header exactly; tests/test_abi.py checks sizeof/offsets
against values compiled from the header."""
import ctypes as C

TW_ABI_VERSION = 7
TW_SCORE_KEEP_WINDOWS = 1
TW_MAX_E = 8
TW_K = 5
TW_MAX_WINDOW = 30
TW_WINDOW_CAP = 31
TW_PARAM_BATCH = 100
TW_PARAM_NBATCHES = 10
TW_WEIGHT_OFFSET = 10000.0
TW_GMM_MAX_COMP = 5
TW_GAUSS_REC = 3
TW_MIX_REC = 21
TW_TERM_ROOT = -1
TW_TERM_LAST = -2
TW_PARAMS_GAUSS_BATCHED = 0
TW_PARAMS_MIXTURE = 1
TW_ASSESS_SCORED, TW_ASSESS_NA, TW_ASSESS_RANGE, TW_ASSESS_CONTAIN, TW_ASSESS_ORDER = 0, 1, 2, 3, 4
TW_ASSESS_NCODES = 5
TW_SKIP_ASSESS_UNDEFINED = 5
TW_SKIP_ASSESS_NCODES = 6

TW_OK = 0
TW_ERR_INVALID, TW_ERR_CUDA, TW_ERR_MWIS_LIMIT, TW_ERR_RANGE_LIMIT, TW_ERR_UNSUPPORTED, TW_ERR_NO_DEVICE, \
    TW_ERR_REFERENCE_UNDEFINED = -1, -2, -3, -4, -5, -6, -7
STATUS = {0: "TW_OK", -1: "TW_ERR_INVALID", -2: "TW_ERR_CUDA", -3: "TW_ERR_MWIS_LIMIT",
          -4: "TW_ERR_RANGE_LIMIT", -5: "TW_ERR_UNSUPPORTED", -6: "TW_ERR_NO_DEVICE",
          -7: "TW_ERR_REFERENCE_UNDEFINED"}

P = C.c_void_p


class TwBatch(C.Structure):
    _fields_ = [
        ("n_problems", C.c_int32), ("n_ep_total", C.c_int32), ("n_term_total", C.c_int32),
        ("reserved0", C.c_int32), ("n_in_total", C.c_int64), ("n_out_total", C.c_int64),
        ("prob_in_off", P), ("prob_ep_off", P), ("prob_tuple_off", P), ("ep_out_off", P),
        ("ep_term_off", P), ("ep_pred_mask", P), ("term_src", P),
        ("in_start", P), ("in_end", P), ("out_start", P), ("out_end", P),
    ]


class TwTimesF64(C.Structure):
    _fields_ = [("in_start", P), ("in_end", P), ("out_start", P), ("out_end", P)]


class TwParams(C.Structure):
    _fields_ = [("mode", C.c_int32), ("reserved0", C.c_int32), ("prob_gauss_off", P),
                ("gauss", P), ("mix", P)]


class TwPassOut(C.Structure):
    _fields_ = [("assign", P), ("mis_rank", P), ("n_cand", P), ("topk_score", P),
                ("topk_idx", P), ("topk_cnt", P), ("counters", P)]


class TwScoreOut(C.Structure):
    _fields_ = [("topk_score", P), ("topk_idx", P), ("topk_cnt", P), ("n_feasible", P), ("cut", P),
                ("used_lo", P), ("used_bits", P), ("used_wide", P), ("flags", C.c_uint32),
                ("reserved0", C.c_uint32)]


class TwSkipDesc(C.Structure):
    _fields_ = [("prob_win_off", P), ("win_start", P), ("prob_cnt_off", P), ("skip_count", P),
                ("prob_pair_off", P), ("pair_gauss", P), ("prob_normalized", P), ("ep_pred_order", P),
                ("out_entry_pos", P), ("out_sorted_of_entry", P)]


class TwSkipOut(C.Structure):
    _fields_ = [("pass_", TwPassOut), ("top2_score", P), ("top2_idx", P), ("top2_cnt", P), ("cut", P)]


class TwTraceKeys(C.Structure):
    _fields_ = [("in_trace", P), ("out_trace", P), ("prob_trace_lo", P), ("prob_trace_n", P),
                ("n_traces", C.c_int32), ("reserved0", C.c_int32)]


def fill(cls, arrays, **values):
    """A `cls` instance built by field name: each pointer field points at `arrays[name]` (a numpy
    array on the host or a torch tensor on the device; NULL when the name is missing or None), a
    nested structure is filled from the same mapping, and the other fields come from `values`."""
    s = cls(**values)
    for name, typ in cls._fields_:
        if typ is P:
            a = arrays.get(name)
            if a is not None:
                setattr(s, name, a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data)
        elif issubclass(typ, C.Structure):
            setattr(s, name, fill(typ, arrays))
    return s


class TwError(RuntimeError):
    def __init__(self, code, where, detail=""):
        self.code = code
        super().__init__(f"{where}: {STATUS.get(code, code)} {detail}".strip())
