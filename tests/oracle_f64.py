"""A second build of the CPU oracle (oracle/tw_oracle.c + its GMM part) with float64 timestamps.

TEST INFRASTRUCTURE ONLY.  The oracle's sources are copied into a temporary directory and only the
declarations that hold timestamps change type (int64_t -> double), so every delay is a plain double
subtraction and every pass-0 mean a sequential double sum of per-element differences, as the reference
computes them on the float start times executor.py --compress_factor > 1 produces.  It shares nothing
with the engine's fixed-point conversion, so engine == this oracle is a real check.  Each replacement
must match exactly once: if the oracle's sources change, the build fails instead of drifting.

    ob = oracle_f64.OracleBatch(hb)      # hb: a float64 HostBatch; the API of oracle.tw_oracle
"""
import ctypes as C
import hashlib
import importlib.util
import os
import re
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
HEADER = os.path.join(ROOT, "include", "traceweaver_b200.h")
SOURCES = ("tw_oracle.c", "tw_oracle.h", "tw_oracle_gmm.c", "tw_oracle_driver.c")

# (old, new, occurrences) in oracle/tw_oracle.c
ORACLE_EDITS = [
    ("const int64_t *is, *ie;", "const double *is, *ie;", 1),
    ("const int64_t *os[TW_MAX_E], *oe[TW_MAX_E];", "const double *os[TW_MAX_E], *oe[TW_MAX_E];", 1),
    ("int64_t exit_t = v->ie[i];", "double exit_t = v->ie[i];", 1),
    ("int64_t st = v->os[s][r->idx[s][h]];", "double st = v->os[s][r->idx[s][h]];", 1),
    ("int64_t x = *(const int64_t*)a, y = *(const int64_t*)b;", "double x = *(const double*)a, y = *(const double*)b;", 1),
    ("static void dist_params(const int64_t* t1, const int64_t* t2,", "static void dist_params(const double* t1, const double* t2,", 1),
    ("int64_t num = 0;", "double num = 0;", 1),
    ("int64_t nn = 0;", "double nn = 0;", 1),
    ("int64_t* in_s = (int64_t*)malloc(sizeof(int64_t)", "double* in_s = (double*)malloc(sizeof(double)", 1),
    ("int64_t* in_e = in_s + n;", "double* in_e = in_s + n;", 1),
    ("memcpy(in_s, v.is, sizeof(int64_t) * (size_t)n); memcpy(in_e, v.ie, sizeof(int64_t) * (size_t)n);",
     "memcpy(in_s, v.is, sizeof(double) * (size_t)n); memcpy(in_e, v.ie, sizeof(double) * (size_t)n);", 1),
    ("qsort(in_s, (size_t)n, sizeof(int64_t), cmp_i64); qsort(in_e, (size_t)n, sizeof(int64_t), cmp_i64);",
     "qsort(in_s, (size_t)n, sizeof(double), cmp_i64); qsort(in_e, (size_t)n, sizeof(double), cmp_i64);", 1),
    ("int64_t* os[TW_MAX_E]; int64_t* oe[TW_MAX_E];", "double* os[TW_MAX_E]; double* oe[TW_MAX_E];", 1),
    ("os[e] = (int64_t*)malloc(sizeof(int64_t) * (size_t)n * 2);", "os[e] = (double*)malloc(sizeof(double) * (size_t)n * 2);", 1),
    ("memcpy(os[e], v.os[e], sizeof(int64_t) * (size_t)n); memcpy(oe[e], v.oe[e], sizeof(int64_t) * (size_t)n);",
     "memcpy(os[e], v.os[e], sizeof(double) * (size_t)n); memcpy(oe[e], v.oe[e], sizeof(double) * (size_t)n);", 1),
    ("qsort(os[e], (size_t)n, sizeof(int64_t), cmp_i64); qsort(oe[e], (size_t)n, sizeof(int64_t), cmp_i64);",
     "qsort(os[e], (size_t)n, sizeof(double), cmp_i64); qsort(oe[e], (size_t)n, sizeof(double), cmp_i64);", 1),
]
# the four span arrays of tw_batch
HEADER_FIELD = re.compile(r"const int64_t\* (in_start|in_end|out_start|out_end);")


def _transform():
    files = {}
    src = open(os.path.join(ORACLE, "tw_oracle.c")).read()
    for old, new, count in ORACLE_EDITS:
        if src.count(old) != count:
            raise RuntimeError(f"oracle_f64: {old!r} occurs {src.count(old)} times in oracle/tw_oracle.c, expected {count}")
        src = src.replace(old, new)
    files["oracle/tw_oracle.c"] = src
    for name in SOURCES[1:]:
        files[f"oracle/{name}"] = open(os.path.join(ORACLE, name)).read()
    hdr, n = HEADER_FIELD.subn(r"const double* \1;", open(HEADER).read())
    if n != 4:
        raise RuntimeError(f"oracle_f64: {n} tw_batch span fields found in the header, expected 4")
    files["include/traceweaver_b200.h"] = hdr
    return files


def build():
    """Compile the float64 oracle into a temporary directory keyed by the sources' hash; returns the .so."""
    files = _transform()
    key = hashlib.sha256("".join(k + v for k, v in sorted(files.items())).encode()).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), f"tw_oracle_f64_{os.getuid()}_{key}")
    so = os.path.join(d, "oracle", "libtw_oracle_f64.so")
    if os.path.exists(so):
        return so
    tmp = tempfile.mkdtemp(prefix="tw_oracle_f64_")
    for rel, text in files.items():
        os.makedirs(os.path.join(tmp, os.path.dirname(rel)), exist_ok=True)
        with open(os.path.join(tmp, rel), "w") as f:
            f.write(text)
    srcs = [os.path.join(tmp, "oracle", s) for s in SOURCES if s.endswith(".c")]
    subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-ffp-contract=off", "-fno-fast-math",
                           "-pthread", "-shared", "-o", os.path.join(tmp, "oracle", "libtw_oracle_f64.so")] + srcs + ["-lm"])
    try:
        os.rename(tmp, d)
    except OSError:          # another process built it first
        pass
    return so if os.path.exists(so) else os.path.join(tmp, "oracle", "libtw_oracle_f64.so")


def _load_frontend():
    """A private copy of oracle/tw_oracle.py (the ctypes front end) bound to the float64 library."""
    spec = importlib.util.spec_from_file_location("tw_oracle_f64_frontend", os.path.join(ORACLE, "tw_oracle.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    lib = C.CDLL(build())
    for name in ("two_params_pass0", "two_score_problem", "two_stitch_problem", "two_delays", "two_windows_from_cuts"):
        getattr(lib, name).restype = C.c_int
    mod._LIB = lib
    return mod


_FRONTEND = _load_frontend()
OracleBatch = _FRONTEND.OracleBatch
gmm_refit = _FRONTEND.gmm_refit
find_assignments = _FRONTEND.find_assignments
