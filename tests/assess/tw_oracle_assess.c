/*
 * tw_oracle_assess.c — the CPU oracle's scoring of a GIVEN assignment.  TEST INFRASTRUCTURE ONLY.
 *
 * Compiled together with the oracle (oracle/tw_oracle.c is included as a whole, so its problem view
 * and score_tuple() — the restatement pinned to the reference's goldens — are reused unchanged) by
 * tests/assess_backends.py, with int64 timestamps or with the float64 edit of tests/oracle_f64.py.
 */
#include "../../oracle/tw_oracle.c"

/* ------------------------------------------------------------------------------------------
 * A GIVEN assignment scored: ScoreAssignmentAsPerInvocationGraph (V1:259-361) of in-span i's
 * tuple after the feasibility checks of DfsTraverseX (V3:328-347).  code[i]: TW_ASSESS_*, the
 * lowest whose condition holds; score[i] NaN unless scored.  prob_sum / prob_count: the scored
 * in-spans' scores added in in-span order, and the in-spans per code.
 * ---------------------------------------------------------------------------------------- */
int two_score_assignments(const tw_batch* b, int p, const tw_params* prm, const int32_t* assign, double* score,
                          uint8_t* code, double* prob_sum, int32_t* prob_count) {
  prob_t v; int rc = view(b, p, &v);
  if (rc) return rc;
  int64_t gauss_base = prm->mode == TW_PARAMS_GAUSS_BATCHED ? prm->prob_gauss_off[p] : 0;
  double sum = 0.0;
  for (int k = 0; k < TW_ASSESS_NCODES; ++k) prob_count[(int64_t)p * TW_ASSESS_NCODES + k] = 0;
  for (int i = 0; i < v.n_in; ++i) {
    int c[TW_MAX_E], na = 0, range = 0, inside = 1, order = 1;
    for (int e = 0; e < v.E; ++e) {
      c[e] = assign[v.tuple_off + (int64_t)e * v.n_in + i];
      if (c[e] == -1) na = 1;
      else if (c[e] < 0 || c[e] >= v.n_out[e]) range = 1;
    }
    if (!na && !range) {
      for (int e = 0; e < v.E; ++e)   /* in.start <= s.start, s.end <= in.end (V3:328-333) */
        if (v.os[e][c[e]] < v.is[i] || v.oe[e][c[e]] > v.ie[i]) inside = 0;
      for (int e = 0; e < v.E; ++e)   /* c_b.end <= c_e.start for every DAG edge b -> e (V3:335-347) */
        for (int q = 0; q < v.E; ++q)
          if ((v.pred[e] >> q & 1) && v.oe[q][c[q]] > v.os[e][c[e]]) order = 0;
    }
    int k = na ? TW_ASSESS_NA : range ? TW_ASSESS_RANGE : !inside ? TW_ASSESS_CONTAIN
          : !order ? TW_ASSESS_ORDER : TW_ASSESS_SCORED;
    int64_t gi = v.in_off + i;
    code[gi] = (uint8_t)k;
    score[gi] = NAN;
    if (k == TW_ASSESS_SCORED) {
      score[gi] = score_tuple(&v, prm, gauss_base, i, c);
      sum += score[gi];
    }
    prob_count[(int64_t)p * TW_ASSESS_NCODES + k]++;
  }
  prob_sum[p] = sum;
  return TW_OK;
}

