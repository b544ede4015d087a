"""Checkers of tw_score_assignments for the tests.  TEST INFRASTRUCTURE ONLY.

    oracle_score(hb, assign, gauss=..., mix=..., float_times=False)   the CPU oracle's scoring code
    emul_score(hb, assign, gauss=..., mix=..., top=None)              the engine's assess_in_span on the CPU

tests/assess/tw_oracle_assess.c extends the oracle (oracle/tw_oracle.c, included as a whole) with the
scoring of a given assignment; float_times=True builds it on the float64 edit of the oracle
(tests/oracle_f64.py).  tests/assess/tw_emul_assess.cpp steps k_assess over the engine's own device
function.  Both compile into a temporary directory keyed by the hash of their sources, so the tree is
never written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle.tw_oracle import OracleBatch, _check, _ptr
from traceweaver_b200 import _abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_SOURCES = ("tw_oracle.c", "tw_oracle.h", "tw_oracle_gmm.c", "tw_oracle_driver.c")
_LIBS = {}


def _read(rel):
    with open(os.path.join(ROOT, rel)) as f:
        return f.read()


def _build(name, files, compile_cmd):
    """Write `files` (relative path -> text) into a fresh directory and run compile_cmd(dir, out) there."""
    key = hashlib.sha256("".join(k + v for k, v in sorted(files.items())).encode()).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), f"tw_assess_{name}_{os.getuid()}_{key}")
    so = os.path.join(d, f"lib{name}.so")
    if not os.path.exists(so):
        tmp = tempfile.mkdtemp(prefix=f"tw_assess_{name}_")
        for rel, text in files.items():
            os.makedirs(os.path.join(tmp, os.path.dirname(rel)), exist_ok=True)
            with open(os.path.join(tmp, rel), "w") as f:
                f.write(text)
        subprocess.check_call(compile_cmd(tmp, os.path.join(tmp, f"lib{name}.so")))
        try:
            os.rename(tmp, d)
        except OSError:          # another process built it first
            pass
        if not os.path.exists(so):
            so = os.path.join(tmp, f"lib{name}.so")
    return C.CDLL(so)


def _oracle_lib(float_times):
    name = "oracle_f64" if float_times else "oracle"
    if name not in _LIBS:
        if float_times:
            import oracle_f64
            files = oracle_f64._transform()
        else:
            files = {f"oracle/{s}": _read(f"oracle/{s}") for s in ORACLE_SOURCES}
            files["include/traceweaver_b200.h"] = _read("include/traceweaver_b200.h")
        files["tests/assess/tw_oracle_assess.c"] = _read("tests/assess/tw_oracle_assess.c")
        cmd = lambda d, out: ["gcc", "-O2", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-ffp-contract=off",
                              "-fno-fast-math", "-pthread", "-shared", "-o", out,
                              os.path.join(d, "tests/assess/tw_oracle_assess.c"),
                              os.path.join(d, "oracle/tw_oracle_gmm.c"), os.path.join(d, "oracle/tw_oracle_driver.c"),
                              "-lm"]
        lib = _build(name, files, cmd)
        lib.two_score_assignments.restype = C.c_int
        _LIBS[name] = lib
    return _LIBS[name]


def _emul_lib():
    if "emul" not in _LIBS:
        files = {rel: _read(rel) for rel in ("traceweaver_b200/csrc/tw_core.cuh", "include/traceweaver_b200.h",
                                             "tests/assess/tw_emul_assess.cpp")}
        cmd = lambda d, out: ["g++", "-O2", "-fPIC", "-std=c++17", "-Wall", "-ffp-contract=off", "-shared", "-x", "c++",
                              "-o", out, os.path.join(d, "tests/assess/tw_emul_assess.cpp"), "-lm"]
        lib = _build("emul", files, cmd)
        lib.twe_assess_problem.restype = C.c_int
        _LIBS["emul"] = lib
    return _LIBS["emul"]


def oracle_score(hb, assign, gauss=None, mix=None, float_times=False):
    """two_score_assignments: score / code per in-span, prob_sum / prob_count per service (scores added in
    in-span order)."""
    ob = OracleBatch(hb)
    n = int(hb.prob_in_off[-1])
    res = dict(score=np.full(n, np.nan), code=np.zeros(n, np.uint8), prob_sum=np.zeros(hb.n_problems),
               prob_count=np.zeros((hb.n_problems, _abi.TW_ASSESS_NCODES), np.int32))
    prm = ob._params_struct(gauss, mix)
    assign = np.ascontiguousarray(assign, np.int32)
    L = _oracle_lib(float_times)
    for p in range(hb.n_problems):
        _check(L.two_score_assignments(C.byref(ob.struct), p, C.byref(prm), _ptr(assign), _ptr(res["score"]),
                                       _ptr(res["code"]), _ptr(res["prob_sum"]), _ptr(res["prob_count"])),
               "score_assignments")
    return res


def emul_score(hb, assign, gauss=None, mix=None, top=None):
    """k_assess stepped on the CPU: score / code (/ margin with `top`, a final top-K) per in-span,
    prob_sum / prob_count per service in the kernels' summation order."""
    ob = OracleBatch(hb)
    n, P = int(hb.prob_in_off[-1]), hb.n_problems
    res = dict(score=np.full(n, -7.0), code=np.full(n, 99, np.uint8), margin=np.full(n, -7.0),
               prob_sum=np.zeros(P), prob_count=np.zeros((P, _abi.TW_ASSESS_NCODES), np.int32))
    prm = ob._params_struct(gauss, mix)
    assign = np.ascontiguousarray(assign, np.int32)
    tk = None
    if top is not None:
        keep = {k: np.ascontiguousarray(top[k]) for k in ("topk_score", "topk_idx", "topk_cnt")}
        tk = _abi.fill(_abi.TwScoreOut, keep)
    L = _emul_lib()
    for p in range(P):
        _check(L.twe_assess_problem(C.byref(ob.struct), p, C.byref(prm), _ptr(assign),
                                    C.byref(tk) if tk is not None else None, _ptr(res["score"]), _ptr(res["code"]),
                                    _ptr(res["margin"]), _ptr(res["prob_sum"]), _ptr(res["prob_count"])),
               "emul.assess")
    if top is None:
        del res["margin"]
    return res
