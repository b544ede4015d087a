"""Checker of tw_skip_score_assignments for the tests.  TEST INFRASTRUCTURE ONLY.

Scores a GIVEN tuple of a cache-mode service with the skip oracle's own scoring code and classifies the
tuples it cannot score.  That code (`primary`, `cost` and `score`, V1:117-139 and :259-361) lives as
closures inside oracle/tw_oracle_skip.py:solve_skip, which stays as it is: `scorer` compiles those three
definitions from the oracle's source, unchanged, into a namespace holding one service's lists and model.

Indices name out spans by their position in the lists as given (the caller's order); -1 is ("NA", "NA"),
any code <= -2 a skip span.  Codes (include/traceweaver_b200.h), the lowest that holds:
    0 scored, 1 NA at some callee, 2 index past the end of its list, 3 a real span not inside the in-span,
    4 c_b.end > c_e.start for a DAG edge b -> e between real spans (the check of the search, V3:335-347),
    5 the reference raises on the tuple (all skips, a chain of skipped ancestors, a missing key)."""
import ast
import inspect
import textwrap

import numpy as np

from oracle import tw_oracle_skip as osk

NCODES = 6
_SCORING = ("primary", "cost", "score")
_CODE = None


def _scoring_code():
    """The oracle's scoring closures, compiled from its source as module-level definitions."""
    global _CODE
    if _CODE is None:
        lines, first = inspect.getsourcelines(osk.solve_skip)
        fn = ast.parse(textwrap.dedent("".join(lines))).body[0]
        defs = [n for n in fn.body if isinstance(n, ast.FunctionDef) and n.name in _SCORING]
        assert [n.name for n in defs] == list(_SCORING), "solve_skip's scoring closures moved"
        mod = ast.Module(body=defs, type_ignores=[])
        ast.increment_lineno(mod, first - 1)
        _CODE = compile(mod, osk.__file__, "exec")
    return _CODE


def scorer(in_start, in_end, out_start, out_end, preds, tab, normalized):
    """score(i, tup) of the oracle for one service: the free names of its closures bound to this service."""
    ns = dict(vars(osk), in_start=in_start, in_end=in_end, out_start=out_start, out_end=out_end, preds=preds,
              tab=tab, normalized=normalized, E=len(out_start))
    exec(_scoring_code(), ns)
    return ns["score"]


def assess(score, i, tup, in_start, in_end, out_start, out_end, preds):
    """(code, score) of in-span i's tuple; score NaN unless code 0.  `score`: a scorer() of the service."""
    if any(c == -1 for c in tup):
        return 1, np.nan
    if any(c >= len(o) for c, o in zip(tup, out_start)):
        return 2, np.nan
    for e, c in enumerate(tup):
        if c >= 0 and (in_start[i] > out_start[e][c] or out_end[e][c] > in_end[i]):
            return 3, np.nan
    for e, c in enumerate(tup):
        if c >= 0 and any(tup[b] >= 0 and out_end[b][tup[b]] > out_start[e][c] for b in preds[e]):
            return 4, np.nan
    try:
        return 0, score(i, list(tup))
    except osk.ReferenceUndefined:
        return 5, np.nan


def assess_service(in_start, in_end, out_start, out_end, preds, assign, tab, normalized):
    """Every in-span of a service: assign [E, n] -> score [n], code [n], service score (in-span order),
    code counts [NCODES]."""
    in_start = [int(x) for x in in_start]
    in_end = [int(x) for x in in_end]
    out_start = [[int(x) for x in o] for o in out_start]
    out_end = [[int(x) for x in o] for o in out_end]
    fn = scorer(in_start, in_end, out_start, out_end, preds, tab, normalized)
    assign = np.asarray(assign)
    n = len(in_start)
    score, code = np.full(n, np.nan), np.zeros(n, np.uint8)
    for i in range(n):
        code[i], score[i] = assess(fn, i, [int(c) for c in assign[:, i]], in_start, in_end, out_start, out_end, preds)
    return dict(score=score, code=code, service_score=float(score[code == 0].sum()),
                service_codes=np.bincount(code, minlength=NCODES))
