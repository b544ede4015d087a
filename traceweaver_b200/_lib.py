"""Loader of libtw_b200.so — the engine's C ABI (include/traceweaver_b200.h).

There is no CPU implementation behind this package: if the shared library is missing or no H100
(sm_90) device is visible, loading / engine creation raises."""
import ctypes as C
import os

from . import _abi

_HERE = os.path.dirname(os.path.abspath(__file__))
# TW_B200_SO: developer override to load a measurement variant of the library (csrc/build.py: build_variant)
SO_PATH = os.environ.get("TW_B200_SO") or os.path.join(_HERE, "libtw_b200.so")
_LIB = None

# every symbol include/traceweaver_b200.h declares
SYMBOLS = {
    "tw_abi_version": (C.c_int, []),
    "tw_last_error": (C.c_char_p, []),
    "tw_device_count": (C.c_int, []),
    "tw_engine_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "tw_engine_destroy": (C.c_int, [C.c_void_p]),
    "tw_batch_validate_host": (C.c_int, [C.POINTER(_abi.TwBatch)]),
    "tw_engine_bind": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwBatch), C.POINTER(_abi.TwBatch), C.c_void_p]),
    "tw_engine_bind_f64": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwBatch), C.POINTER(_abi.TwBatch),
                                     C.POINTER(_abi.TwTimesF64), C.c_void_p]),
    "tw_prepare": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tw_engine_status": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tw_engine_launch_count": (C.c_int64, [C.c_void_p]),
    "tw_engine_tile_stats": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_void_p]),
    "tw_params_pass0": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tw_score_topk": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwParams), C.POINTER(_abi.TwScoreOut), C.c_void_p]),
    "tw_stitch": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwParams), C.c_void_p, C.POINTER(_abi.TwScoreOut),
                            C.POINTER(_abi.TwPassOut), C.c_void_p]),
    "tw_score_assignments": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwParams), C.c_void_p, C.POINTER(_abi.TwScoreOut),
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tw_delays": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tw_gmm_refit": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tw_gmm_stream_draws": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tw_skip_solve": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwBatch), C.POINTER(_abi.TwBatch),
                                C.POINTER(_abi.TwSkipDesc), C.POINTER(_abi.TwSkipOut), C.c_void_p]),
    "tw_skip_score_assignments": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwBatch), C.POINTER(_abi.TwBatch),
                                            C.POINTER(_abi.TwSkipDesc), C.c_void_p, C.POINTER(_abi.TwSkipOut),
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tw_gmm_work": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.c_int]),
    "tw_measure_fp64_peak": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.c_void_p]),
    "tw_ground_truth": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwBatch), C.POINTER(_abi.TwBatch),
                                  C.POINTER(_abi.TwTraceKeys), C.c_void_p, C.c_void_p, C.c_void_p]),
    "tw_find_order": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwBatch), C.POINTER(_abi.TwBatch), C.c_void_p, C.c_void_p,
                                C.c_void_p]),
    "tw_accuracy": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwBatch), C.POINTER(_abi.TwBatch), C.c_void_p, C.c_void_p,
                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                              C.c_void_p]),
    "tw_build_dist_samples": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                        C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tw_assemble_traces": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwBatch), C.POINTER(_abi.TwBatch), C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tw_critical_paths": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwBatch), C.POINTER(_abi.TwBatch),
                                    C.POINTER(_abi.TwTimesF64), C.c_void_p, C.c_void_p, C.c_double,
                                    C.POINTER(_abi.TwCriticalOut), C.c_void_p]),
    "tw_request_confidence": (C.c_int, [C.c_void_p, C.POINTER(_abi.TwBatch), C.POINTER(_abi.TwBatch), C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(_abi.TwScoreOut),
                                        C.POINTER(_abi.TwConfidenceOut), C.c_void_p]),
}


def load():
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(SO_PATH):
        raise ImportError(
            f"{SO_PATH} is missing: build it with `python -m traceweaver_b200.csrc.build` "
            "(nvcc, sm_90a).  traceweaver_b200 has no CPU fallback.")
    lib = C.CDLL(SO_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)       # AttributeError if the ABI and the header drift apart
        fn.restype = res
        fn.argtypes = args
    if lib.tw_abi_version() != _abi.TW_ABI_VERSION:
        raise ImportError("libtw_b200.so ABI version mismatch")
    _LIB = lib
    return lib


def check(rc, where):
    if rc != 0:
        detail = load().tw_last_error().decode(errors="replace")
        raise _abi.TwError(rc, where, detail)
