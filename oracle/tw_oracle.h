/* tw_oracle.h — CPU restatement of the reference hot path.  TEST INFRASTRUCTURE ONLY (see
 * tw_oracle.c).  All pointers are HOST pointers; structs are the product's public ones. */
#ifndef TW_ORACLE_H
#define TW_ORACLE_H
#include <stdint.h>
#include "../include/traceweaver_b200.h"
#ifdef __cplusplus
extern "C" {
#endif
/* ComputeEpPairDistParams3, traceweaver_v3.py:580-646 */
int two_params_pass0(const tw_batch* b, int p, const int64_t* prob_gauss_off, double* gauss);
/* FindTopKAssignments on undeleted lists (v3:1185) + CreateWindows2 cuts (v3:1020-1078) */
int two_score_problem(const tw_batch* b, int p, const tw_params* prm, const tw_score_out* out);
/* hot loop of one pass, v3:1159-1219 */
int two_stitch_problem(const tw_batch* b, int p, const tw_params* prm, const uint8_t* cut,
                       const tw_pass_out* out);
/* a given assignment scored: ScoreAssignmentAsPerInvocationGraph (v1:259-361) after the
 * feasibility checks of DfsTraverseX (v3:328-347) */
int two_assess_problem(const tw_batch* b, int p, const tw_params* prm, const int32_t* assign,
                       double* score, uint8_t* code, double* prob_sum, int32_t* prob_count);
/* durations of ComputeEpPairDistParams5, v3:721-760 */
int two_delays(const tw_batch* b, int p, const int32_t* assign, const int64_t* term_sample_off,
               double* delays, int32_t* counts);
/* window list from cut flags, v3:1056-1076 */
int two_windows_from_cuts(int n, const uint8_t* cut, uint8_t* win_end);
/* sklearn GaussianMixture refit restated (tw_oracle_gmm.c), v3:764-786 */
int two_gmm_refit(int32_t n_terms, const int64_t* term_sample_off, const double* delays,
                  const int32_t* counts, uint32_t seed_select, double* mix_out,
                  int32_t* n_selected_out);
/* the refit with every term's 'diag' BIC per component count and every fit's decisions (tw_oracle_gmm.c) */
int two_gmm_refit_record(int32_t n_terms, const int64_t* term_sample_off, const double* delays,
                         const int32_t* counts, uint32_t seed_select, const uint32_t* rng_skip,
                         double* mix_out, int32_t* n_selected_out, int32_t* max_n_out, double* bic_out,
                         int32_t* rec_out);
/* all problems, both passes, `threads` worker threads (cpu_baseline / --impl reference) */
int two_find_assignments(const tw_batch* b, uint32_t seed_select, int threads,
                         const tw_pass_out* final, const tw_score_out* topk_final,
                         int32_t* n_cand_total, double* mix_out);
#ifdef __cplusplus
}
#endif
#endif
